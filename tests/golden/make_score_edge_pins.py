"""Pins of the scoring edge grid (tests/score_edges.py) from the UNMODIFIED reference (container-only; needs the reference
checkout that oracle/ref_shim.py imports):

    python tests/golden/make_score_edge_pins.py

writes tests/golden/score_edge_pins.npz with, for MoL vector i and RAW vector j,
  mol_bias_i (30,), mol_y_i (n,), mol_nll_i (n,)       utils/distribution.py:16-84, discretized_mix_logistic_loss
                                                      (reduce=False) of each target under the vector's logits
  raw_bias_j (512,), raw_y_j (m,), raw_nll_j (m,)      F.cross_entropy (train_wavernn.py:83, RAW head), the labels by
                                                      the header's rule, as make_score_pins.py computes them
  mol_names, raw_names                               the vectors' names, in order
The arrays depend on the grid and the reference alone: a second run writes identical arrays."""
import sys
from pathlib import Path

import numpy as np
import torch
import torch.nn.functional as F

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))
sys.path.insert(0, str(HERE.parent))

from oracle import ref_shim  # noqa: E402
import score_edges as E  # noqa: E402

F32 = np.float32


def main():
    ref_shim.load_reference()
    from utils.distribution import discretized_mix_logistic_loss
    out = {}
    mol, raw = E.mol_grid(), E.raw_grid()
    for i, (_, bias, y) in enumerate(mol):
        lg = torch.from_numpy(np.repeat(bias[None], y.size, 0))[None]          # (1, n, 30)
        out[f"mol_bias_{i}"], out[f"mol_y_{i}"] = bias, y
        out[f"mol_nll_{i}"] = discretized_mix_logistic_loss(lg, torch.from_numpy(y)[None, :, None],
                                                            reduce=False)[0, :, 0].numpy().astype(F32)
    for j, (_, bias, y) in enumerate(raw):
        labels = np.clip(np.rint((y + F32(1)) * F32(511) * F32(0.5)), 0, 511).astype(np.int64)
        lg = torch.from_numpy(np.repeat(bias[None], y.size, 0))
        out[f"raw_bias_{j}"], out[f"raw_y_{j}"] = bias, y
        out[f"raw_nll_{j}"] = F.cross_entropy(lg, torch.from_numpy(labels), reduction='none').numpy().astype(F32)
    out["mol_names"] = np.array([n for n, _, _ in mol])
    out["raw_names"] = np.array([n for n, _, _ in raw])
    for k, v in out.items():
        if k.endswith(("nll_0", "nll_8")):
            print(k, "finite", bool(np.isfinite(v).all()), "range", float(v.min()), float(v.max()))
    np.savez_compressed(HERE / "score_edge_pins.npz", **out)


if __name__ == "__main__":
    main()
