"""The persistent engine's two tile kernels compute the S1, S2 and S3 chains (K = 512) as (sum over K half 0) + (sum
over K half 1): the small tile (<= 24 folds) stacks both halves in the idle rows of one wgmma chain, the BIG tile (25-64
folds) runs two accumulators.  A fold's samples and logits must therefore not depend on the tile that runs it.

One 40-fold job (a BIG tile), teacher-forced with explicit draws, against folds [f0, f0 + n) run alone for
n = 1, 7, 8, 9, 16, 19, 24, each with its own seg_first and draws: every small-tile row-group count (1, 2, 3 groups, a
group boundary on either side), the headline job's 19 folds and the largest small tile, bit for bit.  The 40-fold run
is also held to the emulation's logit tolerance.  fp16 and bf16, MoL and RAW heads."""
import numpy as np
import pytest

import kernel_jobs as K
from test_gpu_instantiations import Matrix, check_samples, launch, logit_error

pytestmark = pytest.mark.gpu

N_BIG = 40
PARTS = ((39, 1), (3, 7), (8, 8), (30, 9), (12, 16), (21, 19), (16, 24))     # (f0, n)
CASES = [(p, h) for p in ("fp16", "bf16") for h in ("MOL", "RAW")]


@pytest.fixture(scope="module")
def mx():
    m = Matrix()
    yield m
    m.close()


@pytest.mark.parametrize("precision,head", CASES, ids=[f"{p}-{h}" for p, h in CASES])
def test_small_tiles_reproduce_the_big_tile_bit_for_bit(mx, precision, head):
    assert N_BIG > K.SMALL_TILE and all(n <= K.SMALL_TILE and f0 + n <= N_BIG for f0, n in PARTS)
    eng = mx.engine("persistent", precision, head)
    job = mx.job(N_BIG, head, False)
    out, lg, name, grid, launches = launch(eng, job, "rows")
    assert name == f"tcgen05-{precision}" and grid == 128 and launches == 1
    _, emu_lg = mx.emu(precision, N_BIG, head, False)
    err = logit_error(lg, emu_lg, precision, head, N_BIG)
    check_samples(job, out, lg)
    for f0, n in PARTS:
        o, g, _, _, _ = launch(eng, job, "rows", a=f0, b=f0 + n)
        assert np.array_equal(o, out[f0:f0 + n]), ("samples", f0, n)
        assert np.array_equal(g, lg[:, f0:f0 + n]), ("logits", f0, n)
    print(f"persistent {precision} {head}: {N_BIG}-fold BIG tile == small tiles of {[n for _, n in PARTS]} folds; "
          f"max logit error vs emulation {err:.2e}")
