"""Pins of the per-sample training loss (wrnn_score) from the UNMODIFIED reference (container-only; needs the reference
checkout that oracle/ref_shim.py imports):

    python tests/golden/make_score_pins.py

writes tests/golden/score_pins.npz with
  (a) the reference's loss functions on crafted logits and targets -- utils/distribution.py:16-84
      (discretized_mix_logistic_loss, reduce=False) and F.cross_entropy (train_wavernn.py:83, RAW head):
        mol_logits (N, 30), mol_y (N,), mol_nll (N,)        y = +-1, +-0.999 +- 1 ulp, cdf_delta straddling 1e-5,
                                                           log-scales at and below log(1e-14), dominant / flat mixtures
        raw_logits (M, 512), raw_y (M,), raw_nll (M,)      labels 0 and 511, ties, extreme logits
  (b) the shipped checkpoint teacher-forced on the `raw` samples of trained_tacotron.npz: trained_nll (4, 12100).  Each
      fold is fed its rows as generate() folds them -- upsample on the whole padded mel, fold_with_overlap
      (models/fatchord_version.py:293-340; the last fold's rows past the stream are zeros) -- through the layers of
      forward() after its upsample (:131-167); forward itself cannot be called per fold, because it re-upsamples.
  (c) the random-init model (seed 0) on a random mel, unbatched (one fold), teacher-forced on a synthetic waveform:
      rand_mel (80, T), rand_x (n,), rand_nll (n,).
"""
import sys
from pathlib import Path

import numpy as np
import torch
import torch.nn.functional as F

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))
sys.path.insert(0, str(HERE.parent))

from oracle import ref_shim  # noqa: E402
import helpers  # noqa: E402

F32 = np.float32


def crafted_mol(rs):
    """Logits and targets that reach every branch of discretized_mix_logistic_loss."""
    one, p999 = F32(1), F32(0.999)
    ys = [F32(-1), one, p999, -p999, np.nextafter(p999, one), np.nextafter(p999, F32(0)), np.nextafter(-p999, -one),
          np.nextafter(-p999, F32(0)), F32(0), F32(0.5), F32(-0.25)]
    L, Y = [], []
    for y in ys:                                     # generic mixtures at every edge target
        for _ in range(3):
            lg = rs.randn(30).astype(F32)
            lg[10:20] = rs.uniform(-1, 1, 10)
            lg[20:] = rs.uniform(-8, 0, 10)
            L.append(lg); Y.append(y)
    lsm = F32(np.log(1e-14))
    for y in (F32(0.3), F32(-1), F32(1), F32(0.999)):   # log-scales at and below log(1e-14)
        for ls in (lsm, np.nextafter(lsm, F32(0)), F32(-40), F32(-100)):
            lg = rs.randn(30).astype(F32)
            lg[10:20] = y + rs.uniform(-1e-4, 1e-4, 10)
            lg[20:] = ls
            L.append(lg); Y.append(y)
    # cdf_delta straddling 1e-5: a single dominant component whose bin mass sweeps across 1e-5
    for off in np.linspace(0.0, 2.5, 41):
        lg = np.zeros(30, F32)
        lg[0] = 30.0
        lg[10:20] = F32(0.2)
        lg[20:] = F32(-7.0)
        L.append(lg); Y.append(F32(0.2 + off * np.exp(-7.0) * 5))
    for y in (F32(0.1), F32(-0.9), F32(0.99)):        # dominant and flat mixtures
        lg = rs.randn(30).astype(F32); lg[:10] = 0; lg[3] = 60.0
        L.append(lg); Y.append(y)
        lg = rs.randn(30).astype(F32); lg[:10] = 0
        L.append(lg); Y.append(y)
    return np.stack(L).astype(F32), np.array(Y, F32)


def crafted_raw(rs):
    L, Y = [], []
    lab = lambda k: F32(2 * k / 511.0 - 1)           # label_2_float (utils/dataset.py:88)
    for k in (0, 511, 1, 255, 256, 510):
        L.append(rs.randn(512).astype(F32)); Y.append(lab(k))
    lg = np.zeros(512, F32); L.append(lg); Y.append(lab(0))                         # all tied
    lg = np.zeros(512, F32); lg[[7, 300]] = 5.0; L.append(lg); Y.append(lab(300))   # a tie at the top
    lg = np.zeros(512, F32); lg[[7, 300]] = 5.0; L.append(lg); Y.append(lab(7))
    lg = rs.randn(512).astype(F32) * 30; L.append(lg); Y.append(lab(int(np.argmin(lg))))     # extreme logits
    lg = rs.randn(512).astype(F32); lg[511] = 80.0; L.append(lg); Y.append(lab(0))
    lg = rs.randn(512).astype(F32); lg[0] = -80.0; L.append(lg); Y.append(lab(0))
    for y in (F32(-1.2), F32(1.3)):                                                  # clamped labels
        L.append(rs.randn(512).astype(F32)); Y.append(y)
    return np.stack(L).astype(F32), np.array(Y, F32)


def teacher_forced_logits(model, m_up, aux, x_prev):
    """fatchord_version.py:131-167 after `mels, aux = self.upsample(mels)`: m_up (B, S, 80), aux (B, S, 128), x_prev
    (B, S) the previous samples."""
    bsize = x_prev.size(0)
    h1 = torch.zeros(1, bsize, model.rnn_dims)
    h2 = torch.zeros(1, bsize, model.rnn_dims)
    aux_idx = [model.aux_dims * i for i in range(5)]
    a1 = aux[:, :, aux_idx[0]:aux_idx[1]]
    a2 = aux[:, :, aux_idx[1]:aux_idx[2]]
    a3 = aux[:, :, aux_idx[2]:aux_idx[3]]
    a4 = aux[:, :, aux_idx[3]:aux_idx[4]]
    x = torch.cat([x_prev.unsqueeze(-1), m_up, a1], dim=2)
    x = model.I(x)
    res = x
    x, _ = model.rnn1(x, h1)
    x = x + res
    res = x
    x = torch.cat([x, a2], dim=2)
    x, _ = model.rnn2(x, h2)
    x = x + res
    x = torch.cat([x, a3], dim=2)
    x = F.relu(model.fc1(x))
    x = torch.cat([x, a4], dim=2)
    x = F.relu(model.fc2(x))
    return model.fc3(x)


def scored(model, mel, batched, target, overlap, x):
    """The loss of x (B, S) per fold under the rows generate() gives each fold."""
    from utils.distribution import discretized_mix_logistic_loss
    with torch.no_grad():
        m = model.pad_tensor(mel.transpose(1, 2), pad=model.pad, side='both')     # :184-186
        m_up, aux = model.upsample(m.transpose(1, 2))
        if batched:
            m_up = model.fold_with_overlap(m_up, target, overlap)
            aux = model.fold_with_overlap(aux, target, overlap)
        x = torch.as_tensor(x)
        S = x.shape[1]
        x_prev = torch.cat([torch.zeros(x.shape[0], 1), x[:, :-1]], dim=1)
        logits = teacher_forced_logits(model, m_up[:, :S], aux[:, :S], x_prev)
        return discretized_mix_logistic_loss(logits, x.unsqueeze(-1), reduce=False)[:, :, 0].numpy().astype(F32)


def main():
    ref_shim.load_reference()
    from utils.distribution import discretized_mix_logistic_loss
    rs = np.random.RandomState(20261016)
    out = {}
    ml, my = crafted_mol(rs)
    out["mol_logits"], out["mol_y"] = ml, my
    out["mol_nll"] = discretized_mix_logistic_loss(torch.from_numpy(ml)[None], torch.from_numpy(my)[None, :, None],
                                                   reduce=False)[0, :, 0].numpy().astype(F32)
    rl, ry = crafted_raw(rs)
    labels = np.clip(np.rint((ry + F32(1)) * F32(511) * F32(0.5)), 0, 511).astype(np.int64)
    out["raw_logits"], out["raw_y"] = rl, ry
    out["raw_nll"] = F.cross_entropy(torch.from_numpy(rl), torch.from_numpy(labels), reduction='none').numpy().astype(F32)

    g = np.load(HERE / "trained_tacotron.npz")
    model = ref_shim.build_reference_model(seed=0, mode="MOL", pretrained=True)
    model.eval()
    mel = torch.from_numpy(helpers.tacotron_mels()[int(g["sentence"])]).unsqueeze(0)
    out["trained_nll"] = scored(model, mel, True, int(g["target"]), int(g["overlap"]), g["raw"])
    print("trained: mean", out["trained_nll"].mean(), "median", np.median(out["trained_nll"]))

    model = ref_shim.build_reference_model(seed=0, mode="MOL")
    model.eval()
    T, n = 12, 3000
    mel = rs.rand(80, T).astype(F32)
    t = np.arange(n)
    x = (0.6 * np.sin(2 * np.pi * t / 97.0) + 0.05 * rs.randn(n)).astype(F32)
    x[::250] = 1.0; x[125::250] = -1.0                 # the edge branches
    x = np.clip(x, -1, 1).astype(F32)
    out["rand_mel"], out["rand_x"] = mel, x
    out["rand_nll"] = scored(model, torch.from_numpy(mel)[None], False, 0, 0, x[None])[0]
    print("random init: mean", out["rand_nll"].mean())
    np.savez_compressed(HERE / "score_pins.npz", **out)


if __name__ == "__main__":
    main()
