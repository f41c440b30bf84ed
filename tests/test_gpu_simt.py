"""The SIMT engine (wrnn_simt.cu) against the engine-arithmetic emulation, one test per arithmetic path:

  wrnn_simt_kernel<T>   T = float | __half | __nv_bfloat16   x   MoL | RAW head (chosen at run time)   (6)

The fp32 handle is made on ENGINE_AUTO, which serves every fp32 job with this engine; the others on ENGINE_SIMT.  The
jobs are those of the tensor-core matrix (tests/kernel_jobs.py: stride 271 against the 275 hop, steps < seg_len,
seg_first != 0, the last fold past the stream, fold tables with short and mid-frame windows), at 24, 25, 73, 17 and 33
folds: 1, 1, 3, 1 and 2 of the kernel's 32-fold tiles, the last one ragged.  Each runs strided and with fold tables, on
materialised rows (the engine takes no frame-rate tensors; that refusal is checked once).

Checks: the engine that ran (name, grid, one launch per job); logits against contract.generate_segments at the
handle's precision within kernel_jobs.LOGIT_TOL; fp32 also against wavernn_oracle.generate_segments (the reference's
unfolded order) within kernel_jobs.ORACLE_TOL; fp16 / bf16 also closer, on the mean logit error, to their own
precision's emulation than to the other's (kernel_jobs.ROUNDING_SEPARATION); samples against the kernel's own logits
under the libm error model; the 73-fold job bit for bit equal to its folds run as [0, 32) + [32, 64) + [64, 73) and as
[0, 1) + [1, 73).  That last check holds by construction: lane f of a tile accumulates fold f alone, over the same k
order whatever its lane or tile (gemv_tile, out_row), and the RAW sampler gives each fold one warp that strides the
classes the same way for every fold, so nothing a fold computes depends on where in the launch it sits.
Run on a GPU: pytest -m gpu -s (one line per path)."""
import numpy as np
import pytest
import torch

import helpers
import kernel_jobs as K
from oracle import wavernn_oracle as O
from test_gpu_instantiations import Matrix, check_samples, launch, logit_error
from test_gpu_sampling import LIBM
from wavernn_b200 import cabi

pytestmark = pytest.mark.gpu

PATHS = [(p, h) for p in ("fp32", "fp16", "bf16") for h in ("MOL", "RAW")]
FOLDS = (24, 25, 73, 17, 33)
FT = 32                                   # folds per SIMT tile
OTHER = {"fp16": "bf16", "bf16": "fp16"}
SPLITS = (((0, 32), (32, 64), (64, 73)),  # the three tiles as jobs of their own
          ((0, 1), (1, 73)))              # every fold of [1, 73) one lane lower in its tile


@pytest.fixture(scope="module")
def sm():
    m = Matrix()
    yield m
    m.close()


def simt_engine(sm, precision, head):
    key = ("simt", precision, head)
    if key not in sm.engines:
        m = sm.model(head)[0]
        sm.engines[key] = cabi.Engine(m.hot_state(), n_classes=m.n_classes, mode=head, precision=precision,
                                      engine="auto" if precision == "fp32" else "simt", device=0)
    return sm.engines[key]


def test_the_jobs_cover_the_tiles():
    tiles = [-(-n // FT) for n in FOLDS]
    assert tiles == [1, 1, 3, 1, 2] and 73 % FT and 33 % FT
    assert sorted(FOLDS) == sorted({n for n, _ in K.all_jobs()})


@pytest.mark.parametrize("precision,head", PATHS, ids=[f"simt-{p}-{h}" for p, h in PATHS])
def test_simt_path(sm, precision, head):
    eng = simt_engine(sm, precision, head)
    w = sm.model(head)[1]

    def run(job, **kw):
        out, lg, name, grid, launches = launch(eng, job, "rows", **kw)
        assert name == f"simt-{precision}" and grid == 128 and launches == 1, (name, grid, launches)
        return out, lg

    with pytest.raises(cabi.EngineError, match=f"outside the envelope of engine 'simt-{precision}'"):
        launch(eng, sm.job(24, head, True), "frames")
    errs, oracle_errs, own, other = [], [], [], []
    for n in FOLDS:
        for tables in (False, True):
            job = sm.job(n, head, tables)
            _, emu_lg = sm.emu(precision, n, head, tables)
            out, lg = run(job)
            errs.append(logit_error(lg, emu_lg, precision, head, (n, tables)))
            check_samples(job, out, lg, acc=LIBM)
            if precision == "fp32":
                _, ref_lg = K.emulate_oracle(w, job)
                oracle_errs.append(float(np.abs(lg.astype(np.float64) - ref_lg).max()))
                assert oracle_errs[-1] <= K.ORACLE_TOL[head], ("reference order", n, tables, oracle_errs[-1])
            else:
                _, other_lg = sm.emu(OTHER[precision], n, head, tables)
                own.append(np.abs(lg.astype(np.float64) - emu_lg).ravel())
                other.append(np.abs(lg.astype(np.float64) - other_lg).ravel())
            if n == 73:
                for split in SPLITS:
                    parts = [run(job, a=a, b=b) for a, b in split]
                    assert np.array_equal(out, np.concatenate([p[0] for p in parts], 0)), ("samples", split, tables)
                    assert np.array_equal(lg, np.concatenate([p[1] for p in parts], 1)), ("logits", split, tables)
    line = (f"simt {precision} {head}: max logit error vs emulation {max(errs):.2e} "
            f"(tolerance {K.LOGIT_TOL[(precision, head)]:.1e})")
    if precision == "fp32":
        line += f"; vs the reference order {max(oracle_errs):.2e} (bound {K.ORACLE_TOL[head]:.1e})"
    else:
        m_own, m_other = float(np.concatenate(own).mean()), float(np.concatenate(other).mean())
        line += f"; mean error vs {precision} emulation {m_own:.2e}, vs {OTHER[precision]} {m_other:.2e}"
        assert m_own <= m_other / K.ROUNDING_SEPARATION, (m_own, m_other)
    print(line)
