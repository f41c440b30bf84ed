"""Host-side pieces of wrnn_vocode, checked without a device through the library's test hooks: the ABI structs against
the header, fold geometry, the float64 epilogue tables, the 5-tap interpolation table and the folded MelResNet."""
import ctypes
import math
import subprocess
import sys

import numpy as np
import pytest
import torch

import helpers
from wavernn_b200 import cabi
from wavernn_b200.sharding import fold_geometry, unbatched_geometry

ROOT = helpers.GOLDEN.parent.parent


@pytest.fixture(scope="module")
def lib():
    if not cabi.is_built():
        import __graft_entry__ as g
        g.build()
    return cabi.load()


def test_struct_layouts_match_header(tmp_path):
    """The ctypes mirrors against offsetof / sizeof of include/wavernn_b200.h, as the host C compiler lays them out."""
    fields = {"wrnn_tensor": (cabi.WrnnTensor, ("name", "data", "numel")),
              "wrnn_upsample_cfg": (cabi.WrnnUpsampleCfg, ("compute_dims", "res_out_dims", "res_blocks", "pad",
                                                           "n_factors", "factors", "hop_length")),
              "wrnn_vocode_job": (cabi.WrnnVocodeJob, ("mel", "T", "batched", "target", "overlap", "mu_law",
                                                       "philox_seed", "wav"))}
    lines = ["#include <stddef.h>", "#include <stdio.h>", '#include "wavernn_b200.h"', "int main(void) {"]
    for st, (_, names) in fields.items():
        lines.append(f'  printf("{st} %zu\\n", sizeof({st}));')
        lines += [f'  printf("{st}.{n} %zu\\n", offsetof({st}, {n}));' for n in names]
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-std=c99", "-I", str(ROOT / "include"), "-o", str(exe), str(src)], check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    for st, (cls, names) in fields.items():
        assert int(got[st]) == ctypes.sizeof(cls), st
        for n in names:
            assert int(got[f"{st}.{n}"]) == getattr(cls, n).offset, (st, n)
    assert ctypes.sizeof(cabi.WrnnTensor) == 24 and ctypes.sizeof(cabi.WrnnUpsampleCfg) == 40
    assert ctypes.sizeof(cabi.WrnnVocodeJob) == 48 and cabi.WrnnVocodeJob.philox_seed.offset == 32


def test_fold_geometry_matches_sharding(lib):
    out = (ctypes.c_int64 * 5)()
    n = 0
    for T in (21, 22, 26, 37, 100, 800, 1234):
        L = T * 275
        for target, overlap in ((2200, 220), (11000, 550), (1, 1), (275, 275), (5775, 1), (L, 1), (L - 1, 1), (7, 3000),
                                (3000, L), (L // 3, 100), (L // 3 + 1, 99)):
            geo = fold_geometry(L, target, overlap)
            assert lib.wrnn_debug_fold_geometry(L, 1, target, overlap, out) == 0
            assert tuple(out) == (geo.n_seg, geo.seg_len, geo.seg_stride, geo.overlap, geo.padded_len), (L, target, overlap)
            n += geo.padded_len != L
        geo = unbatched_geometry(L)
        assert lib.wrnn_debug_fold_geometry(L, 0, 11000, 550, out) == 0
        assert tuple(out) == (geo.n_seg, geo.seg_len, geo.seg_stride, geo.overlap, geo.padded_len)
    assert n > 10        # padded last folds are part of the sweep


def _c_tables(lib, overlap, mu_law, n_classes, hop):
    fi, fo = np.empty(overlap), np.empty(overlap)
    mu, tail = np.empty(n_classes), np.empty(20 * hop)
    p = lambda a: a.ctypes.data if a.size else None
    assert lib.wrnn_debug_epilogue_tables(overlap, int(mu_law), n_classes, hop, p(fi), p(fo), p(mu), p(tail)) == 0
    return fi, fo, (mu if mu_law else None), tail


@pytest.mark.parametrize("overlap", [1, 2, 3, 220, 550, 551, 1000])
def test_fade_and_tail_tables_are_bit_identical(lib, overlap):
    m = helpers.make_model(0, "RAW")
    geo = fold_geometry(26 * 275, 2200, overlap)
    tabs = m._epilogue_tables(geo, True, False, torch.device("cpu"))
    fi, fo, _, tail = _c_tables(lib, overlap, False, 512, 275)
    assert np.array_equal(fi, tabs["fade_in"].numpy()) and np.array_equal(fo, tabs["fade_out"].numpy())
    assert np.array_equal(tail, tabs["tail"].numpy())
    for hop in (1, 2, 100, 256):        # the fade-out alone, other hops
        assert np.array_equal(_c_tables(lib, 0, False, 512, hop)[3], np.linspace(1, 0, 20 * hop))


def test_mu_law_table(lib):
    """decode_mu_law of the fp32 class values.  The library evaluates pow with the C library's pow, which is what numpy's
    scalar loop calls; so the table is bit-identical to the reference expression evaluated that way.  numpy builds that
    dispatch np.power to a vectorised (AVX-512) pow may differ from it in the last bit of a few entries."""
    m = helpers.make_model(0, "RAW")
    geo = fold_geometry(26 * 275, 2200, 220)
    ref = m._epilogue_tables(geo, True, True, torch.device("cpu"))["mu"].numpy()
    mu = _c_tables(lib, 220, True, 512, 275)[2]
    n = 512
    x = (np.float32(2) * np.arange(n, dtype=np.float32) / np.float32(n - 1) - np.float32(1)).astype(np.float64)
    scalar = np.array([np.sign(v) / (n - 1) * (math.pow(n, abs(v)) - 1) for v in x])
    assert np.array_equal(mu, scalar)
    pw_np, pw_c = np.power(np.float64(n), np.abs(x)), np.array([math.pow(n, abs(v)) for v in x])
    ulps = np.abs(pw_np.view(np.int64) - pw_c.view(np.int64))
    print(f"mu-law table: {int((mu != ref).sum())} of {n} entries differ from numpy's; its np.power differs from pow "
          f"by {int(ulps.max())} ulp at most")
    assert ulps.max() <= 1
    assert np.all(np.abs(mu - ref) <= np.spacing(pw_c) / (n - 1))


def test_every_raw_label_is_recovered_from_the_sample_the_kernels_write():
    """Host mirror of wrnn_epilogue's label recovery for the mu-law table, in float32 as the kernel evaluates it:
    __float2int_rn((x + 1) * (0.5 * (n - 1))) returns k for the sample x = 2k / (n - 1) - 1 that the RAW samplers of
    wrnn_tc.cu / wrnn_simt.cu / wrnn_stream.cu write for class k (`2.0f * (float)k / ((float)n - 1.0f) - 1.0f`), for
    every k < 512.  np.rint rounds half to even, as __float2int_rn does."""
    n = 512
    f = np.float32
    k = np.arange(n)
    x = f(2) * k.astype(f) / (f(n) - f(1)) - f(1)
    assert x.dtype == f and x[0] == -1 and x[-1] == 1 and x[(n - 1) // 2 + 1] > 0 > x[(n - 1) // 2]
    y = (x + f(1)) * (f(0.5) * f(n - 1))
    assert y.dtype == f
    lbl = np.rint(y).astype(np.int64)
    assert np.array_equal(lbl, k), k[lbl != k]
    print(f"RAW labels: largest distance of (x + 1) (n - 1) / 2 from its label {np.abs(y.astype(np.float64) - k).max():.2e}")


# ---------------------------------------------------------------------------------------------------- the upsampler
def _hook(lib, state_dict, **kw):
    cfg = cabi.upsample_cfg(**kw)
    arr, keep = cabi.tensor_list(state_dict)
    blen = ctypes.c_uint64()
    rc = lib.wrnn_debug_upsampler(ctypes.byref(cfg), arr, len(arr), None, ctypes.byref(blen), None)
    if rc != 0:
        return rc, lib.wrnn_last_error().decode(), None, None
    blob, taps = np.empty(blen.value), np.empty(kw.get("hop_length", 275) * 5)
    assert lib.wrnn_debug_upsampler(ctypes.byref(cfg), arr, len(arr), blob.ctypes.data, ctypes.byref(blen), taps.ctypes.data) == 0
    del keep
    return 0, "", blob, taps.reshape(-1, 5)


def _model(pad=2, factors=(5, 5, 11), hop=275, seed=0):
    import contextlib
    import io
    from wavernn_b200 import WaveRNN
    torch.manual_seed(seed)
    kw = dict(helpers.CTOR, pad=pad, upsample_factors=factors, hop_length=hop, rnn_dims=32, fc_dims=32)
    with contextlib.redirect_stdout(io.StringIO()):
        return WaveRNN(mode="MOL", **kw)


def test_tap_table_matches_upsample_taps(lib):
    m = helpers.make_model(0, "MOL")
    rc, msg, _, taps = _hook(lib, m.state_dict())
    assert rc == 0, msg
    ref = m.upsample_taps(torch.device("cpu")).numpy().astype(np.float64)
    err = np.abs(taps - ref).max()
    print(f"tap table: max |C - torch| = {err:.3e} (largest tap {np.abs(ref).max():.3e})")
    assert err <= 2.0 ** -20 * np.abs(ref).max()


@pytest.mark.parametrize("pad,factors,hop", [(2, (5, 5, 11), 275), (1, (5, 5, 11), 275), (3, (5, 5, 11), 275),
                                             (2, (5, 5, 11), 300), (2, (4, 4, 16), 256), (2, (1, 5, 55), 275),
                                             (2, (3,), 3), (2, (2, 3, 4, 5), 120), (2, (11, 5, 5), 275), (2, (2, 2), 4)])
def test_same_geometries_as_kernel_conditioning(lib, pad, factors, hop):
    m = _model(pad, factors, hop)
    ok = m._kernel_conditioning_ok()
    rc, msg, _, taps = _hook(lib, m.state_dict(), pad=pad, upsample_factors=factors, hop_length=hop)
    assert (rc == 0) == ok, (msg, ok)
    if ok:
        ref = m.upsample_taps(torch.device("cpu")).numpy()
        assert np.abs(taps - ref).max() <= 2.0 ** -20 * np.abs(ref).max()
    else:
        assert rc == cabi.WRNN_E_INVALID and ("5-tap" in msg)


def _randomise_batch_norms(m, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for mod in m.upsample.resnet.modules():
            if isinstance(mod, torch.nn.BatchNorm1d):
                mod.weight.uniform_(0.5, 1.5, generator=g)
                mod.bias.uniform_(-0.3, 0.3, generator=g)
                mod.running_mean.uniform_(-0.5, 0.5, generator=g)
                mod.running_var.uniform_(0.2, 2.0, generator=g)


def _folded_forward(blob, mel, R):
    """MelResNet in float64 from the hook's folded parameters (layout of wrnn_cond.h): mel (80, T) -> (T, 128)."""
    T = mel.shape[1]
    o = 0

    def take(n, shape):
        nonlocal o
        a = blob[o:o + n].reshape(shape)
        o += n
        return a
    melp = np.pad(mel.astype(np.float64), ((0, 0), (2, 2)))
    cols = np.stack([melp[:, j:j + T] for j in range(5)], axis=1).reshape(400, T)    # k = c*5 + j
    W, b = take(400 * 128, (400, 128)), take(128, (128,))
    x = np.maximum(W.T @ cols + b[:, None], 0)
    for _ in range(R):
        W1, b1 = take(128 * 128, (128, 128)), take(128, (128,))
        W2, b2 = take(128 * 128, (128, 128)), take(128, (128,))
        y = np.maximum(W1.T @ x + b1[:, None], 0)
        x = W2.T @ y + b2[:, None] + x
    W, b = take(128 * 128, (128, 128)), take(128, (128,))
    assert o == blob.size
    return (W.T @ x + b[:, None]).T


@pytest.mark.parametrize("weights", ["random", "checkpoint"])
def test_folded_weights_reproduce_the_module(lib, weights):
    m = helpers.make_model(0, "MOL")
    if weights == "checkpoint":
        m.load_state_dict(helpers.pretrained_state_dict())
    else:
        _randomise_batch_norms(m, 7)
    rc, msg, blob, _ = _hook(lib, m.state_dict())
    assert rc == 0, msg
    net = m.upsample.resnet.double().eval()
    for T in (21, 64, 97):
        mel = helpers.make_mel(T, seed=T)[0].numpy()
        with torch.no_grad():
            ref = net(torch.from_numpy(np.pad(mel.astype(np.float64), ((0, 0), (2, 2))))[None])[0].numpy().T
        got = _folded_forward(blob, mel, 10)
        rel = np.abs(got - ref).max() / np.abs(ref).max()
        assert rel <= 1e-12, (T, rel)


def test_upsampler_refusals_name_the_key(lib):
    sd = helpers.make_model(0, "MOL").state_dict()
    up = {k: v for k, v in sd.items() if k.startswith("upsample.")}
    assert _hook(lib, sd)[0] == 0                          # the whole state_dict: non-upsample keys are ignored
    k = "upsample.resnet.layers.3.batch_norm2.running_var"
    rc, msg, *_ = _hook(lib, {kk: v for kk, v in up.items() if kk != k})
    assert rc == cabi.WRNN_E_INVALID and "missing key" in msg and k in msg
    rc, msg, *_ = _hook(lib, dict(up, **{"upsample.resnet.layers.10.conv1.weight": up["upsample.resnet.layers.0.conv1.weight"]}))
    assert rc == cabi.WRNN_E_INVALID and "upsample.resnet.layers.10.conv1.weight" in msg
    k = "upsample.resnet.conv_in.weight"
    rc, msg, *_ = _hook(lib, dict(up, **{k: up[k][:, :, :4]}))
    assert rc == cabi.WRNN_E_INVALID and k in msg and "51200" in msg
    rc, msg, *_ = _hook(lib, up, compute_dims=256)
    assert rc == cabi.WRNN_E_INVALID and "unsupported dims" in msg
    rc, msg, *_ = _hook(lib, up, res_out_dims=64)
    assert rc == cabi.WRNN_E_INVALID and "unsupported dims" in msg
    rc, msg, *_ = _hook(lib, up, res_blocks=9)               # one block too few: its tensors are unexpected keys
    assert rc == cabi.WRNN_E_INVALID and "upsample.resnet.layers.9." in msg
    # repeated key
    cfg = cabi.upsample_cfg()
    arr, keep = cabi.tensor_list(up)
    arr2 = (cabi.WrnnTensor * (len(arr) + 1))(*arr, arr[0])
    assert lib.wrnn_debug_upsampler(ctypes.byref(cfg), arr2, len(arr2), None, None, None) == cabi.WRNN_E_INVALID
    assert b"repeated key: upsample.resnet.conv_in.weight" in lib.wrnn_last_error()
    del keep


def test_vocode_refuses_null_handle(lib):
    job = cabi.WrnnVocodeJob()
    assert lib.wrnn_vocode(None, ctypes.byref(job), None) == cabi.WRNN_E_INVALID
    assert lib.wrnn_vocode_host(None, ctypes.byref(job)) == cabi.WRNN_E_INVALID
    assert lib.wrnn_attach_upsampler(None, None, None, 0) == cabi.WRNN_E_INVALID
    assert lib.wrnn_conditioning_frames(None, None, 0, None, None, None, None) == cabi.WRNN_E_INVALID


if __name__ == "__main__":
    sys.exit(pytest.main([__file__, "-v", "-s"]))
