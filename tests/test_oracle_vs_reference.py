"""Pins of the oracle, the CPU timing port and the module against the UNMODIFIED reference, through fixtures the
reference itself produced (tests/golden/make_golden.py -> mol_batched.npz, tests/golden/make_reference_pins.py ->
reference_pins.npz)."""
import numpy as np
import pytest
import torch

import helpers
from oracle import torch_port
from oracle import wavernn_oracle as O


@pytest.fixture(scope="module")
def pins():
    return helpers.load_golden("reference_pins.npz")


def test_oracle_tracks_reference_with_pretrained_weights(pins):
    """Trained weights make the sampler chaotic (SURVEY 7.2): agreement is a PREFIX property."""
    model = helpers.make_model(0, "MOL")
    model.load_state_dict(helpers.pretrained_state_dict(), strict=False)
    model.eval()
    sd = helpers.state_numpy(model)
    mel = helpers.make_mel(30, 0)
    head, raw_std = pins["pretrained_raw_head"], float(pins["pretrained_raw_std"])      # reference: first 1,000 steps, std
    U = helpers.replay_uniforms(1234, 3300, 3)
    wav, pre = O.generate(O.hot_weights(sd), sd, mel[0].numpy(), batched=True, target=2750, overlap=275,
                          uniforms=U, return_pre=True)
    assert np.abs(pre[:, :1000] - head).max() < 1e-4
    assert abs(pre.std() - raw_std) < 0.2 * raw_std


def test_torch_port_reproduces_reference_samples():
    g = helpers.load_golden("mol_batched.npz")
    model = helpers.make_model(0, "MOL")
    model.eval()
    mel = helpers.make_mel(30, 0)
    with torch.no_grad():
        mp = model.pad_tensor(mel.transpose(1, 2), pad=2, side="both").transpose(1, 2)
        m_up, aux = model.upsample(mp)
        mf, af = model.fold_with_overlap(m_up, 2750, 275), model.fold_with_overlap(aux, 2750, 275)
    torch.manual_seed(1234)
    out, _ = torch_port.generate_segments_torch({k: v.detach() for k, v in model.state_dict().items()}, mf, af)
    np.testing.assert_array_equal(out, g["raw"])


def test_dropin_class_loads_pretrained_checkpoint():
    ours = helpers.make_model(0, "MOL")
    missing = ours.load_state_dict(helpers.pretrained_state_dict(), strict=False)
    assert not missing.missing_keys and not missing.unexpected_keys
    assert ours.get_step() == 797232


@pytest.mark.parametrize("mode", ["MOL", "RAW"])
def test_training_forward_equals_reference_forward(mode, pins):
    """SURVEY 8f-4: `WaveRNN.forward(x, mels)` (reference :131-167, what train_wavernn.py:91-155 calls) on the reference's
    seed-0 weights -- eval mode and train mode (BatchNorm batch statistics, running-stat updates, `step` counter) -- and
    the gradients of the training loss, against the reference's values (a fixed sample of every output and gradient)."""
    ours = helpers.make_model(1, mode)                     # different init: everything must come from the state_dict
    ours.load_state_dict(helpers.make_model(0, mode).state_dict())
    torch.manual_seed(5)
    mels = torch.rand(3, 80, 12 + 4)                       # (B, 80, T + 2*pad)
    x = torch.rand(3, 12 * 275) * 2 - 1                    # (B, T*hop)
    for train in (False, True):
        ours.train(train)
        b = ours(x, mels)
        assert b.shape == (3, 12 * 275, 30 if mode == "MOL" else 512)
        y = b.detach().numpy().ravel()
        want = pins[f"fwd_{mode}_{int(train)}_val"]
        got = y[helpers.sample_index(y.size, int(pins["n_out"]), 1 + train)]
        assert np.array_equal(got, want) or np.abs(got - want).max() <= 1e-6
    assert ours.get_step() == int(pins[f"fwd_{mode}_step"])
    sb = ours.state_dict()
    stats = [k for k in sb if "running" in k or "num_batches" in k]
    assert stats and all(f"fwd_{mode}_state_{k}" in pins.files for k in stats)
    for k in stats:                                        # BatchNorm running statistics moved identically
        np.testing.assert_allclose(sb[k].double().numpy(), pins[f"fwd_{mode}_state_{k}"].astype(np.float64), rtol=0, atol=1e-6, err_msg=k)
    # gradients of the training loss flow through the same parameters
    ours.zero_grad()
    ours(x, mels).square().mean().backward()
    names = [k for k, _ in ours.named_parameters()]
    assert sorted(names) == sorted(f[len(f"grad_{mode}_"):-len("_val")] for f in pins.files
                                   if f.startswith(f"grad_{mode}_") and f.endswith("_val"))
    for i, (k, p) in enumerate(ours.named_parameters()):
        g = p.grad.numpy().ravel()
        got = g[helpers.sample_index(g.size, int(pins["n_grad"]), 100 + i)]
        np.testing.assert_allclose(got, pins[f"grad_{mode}_{k}_val"], rtol=1e-4, atol=1e-7, err_msg=k)
