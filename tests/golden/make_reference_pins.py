"""Generates tests/golden/reference_pins.npz from the UNMODIFIED reference (imported through oracle/ref_shim.py), for
tests/test_oracle_vs_reference.py and the public-surface check of tests/test_dropin_api.py.  Run where a checkout of
the reference is available (located by oracle/ref_shim.py, WAVERNN_REFERENCE):

    python tests/golden/make_reference_pins.py

Stored: the first 1,000 steps and the standard deviation of the reference's samples with its shipped checkpoint
(batched 2750 / 275, seed 1234, make_mel(30, 0)); for `WaveRNN.forward` in eval and train mode a fixed seeded sample of
the outputs, the BatchNorm running statistics and step counter after both calls, and a fixed seeded sample of every
parameter's gradient of the training loss; the parameter names of the public methods.  The sample indices are not
stored: tests regenerate them with `helpers.sample_index` from the seeds used here.  Samples keep the file small (the
full RAW forward output is 20 MB).
"""
import inspect
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))
sys.path.insert(0, str(HERE.parent))

from oracle import ref_shim  # noqa: E402
import helpers  # noqa: E402

N_OUT = 2048          # sampled entries of each forward output
N_GRAD = 32           # sampled entries of each parameter's gradient
METHODS = ("forward", "generate", "get_gru_cell", "pad_tensor", "fold_with_overlap", "xfade_and_unfold", "get_step", "log",
           "load", "save", "num_params", "gen_display")


def forward_inputs():
    torch.manual_seed(5)
    mels = torch.rand(3, 80, 12 + 4)                       # (B, 80, T + 2*pad)
    x = torch.rand(3, 12 * 275) * 2 - 1                    # (B, T*hop)
    return x, mels


def main():
    ref = ref_shim.load_reference()
    out = {}
    # pretrained checkpoint, batched generate
    model = ref_shim.build_reference_model(seed=0, mode="MOL", pretrained=True)
    model.eval()
    r = ref_shim.ref_generate(model, helpers.make_mel(30, 0), True, 2750, 275, seed=1234)
    out["pretrained_raw_head"] = r["raw"][:, :1000].astype(np.float32)
    out["pretrained_raw_std"] = np.float64(r["raw"].std())
    # training forward, eval then train mode, and the gradients of the training loss
    for mode in ("MOL", "RAW"):
        m = ref_shim.build_reference_model(seed=0, mode=mode)
        x, mels = forward_inputs()
        for train in (False, True):
            m.train(train)
            y = m(x, mels).detach().numpy().ravel()
            out[f"fwd_{mode}_{int(train)}_val"] = y[helpers.sample_index(y.size, N_OUT, 1 + train)].astype(np.float32)
        out[f"fwd_{mode}_step"] = np.int64(m.get_step())
        for k, v in m.state_dict().items():
            if "running" in k or "num_batches" in k:
                out[f"fwd_{mode}_state_{k}"] = v.detach().numpy().copy()
        m.zero_grad()
        m(x, mels).square().mean().backward()
        for i, (k, p) in enumerate(m.named_parameters()):
            g = p.grad.detach().numpy().ravel()
            out[f"grad_{mode}_{k}_val"] = g[helpers.sample_index(g.size, N_GRAD, 100 + i)].astype(np.float32)
    # public surface
    for name in METHODS + ("__init__",):
        out[f"sig_{name}"] = np.array(list(inspect.signature(getattr(ref.WaveRNN, name)).parameters))
    out["n_out"], out["n_grad"] = np.int64(N_OUT), np.int64(N_GRAD)
    np.savez_compressed(HERE / "reference_pins.npz", **out)
    print("wrote reference_pins.npz,", len(out), "arrays")


if __name__ == "__main__":
    main()
