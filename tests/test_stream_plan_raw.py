"""The stream engine's step program for the 9-bit RAW head (wavernn_b200/csrc/wrnn_stream_plan.h, n_classes == 512),
checked WITHOUT a GPU, like tests/test_stream_plan.py does for the MoL head: the library exports the plan
(wrnn_debug_stream_plan with cfg.mode == RAW), and numpy interprets it the way the kernel's consumer warps do.

fc3 is four 128-class unit blocks, each laid out like an fc1 / fc2 block (four owners, each its K quarter into its
own partial accumulator).  The kernel (wrnn_stream.cu, RAW) reduces every block to one (score, class) per fold with
score = logit - log e, e the class's Exp(1) draw; the pick is the best score, ties to the lowest class.  The cluster
form runs fc3 block r in rank r; every rank writes its candidate into every rank's table and reduces the same four."""
import ctypes as C

import numpy as np
import pytest

import helpers
from oracle import contract as CT
from oracle import philox as P
from oracle import wavernn_oracle as O
from test_stream_plan import decode_tile, sig
from wavernn_b200 import cabi

H, CDIM, NB, NCLS = 512, 208, 4, 512
B_COND, B_H1PREV, B_H1NEW, B_H2, B_Y1, B_Y2, B_NONE = 0, 1, 2, 3, 4, 5, 0xFF
W_NONE, W_COND, W_H1NEW, W_H2NEW, W_Y1, W_Y2 = range(6)
F32 = np.float32

CHUNK = np.dtype([("size16", "<u2"), ("a_off16", "<u2"), ("acc", "u1"), ("nk", "u1"), ("b_buf", "u1"), ("b_buf2", "u1"), ("k0", "<u2"),
                  ("flags", "u1"), ("wait_b", "u1"), ("wait_acc", "u1"), ("commit", "u1"), ("owner", "u1"), ("phase", "u1")])

pytestmark = pytest.mark.skipif(not cabi.is_built(), reason="library not built")


def get_plan_raw(sd, precision="fp16", only_block=-1):
    lib = cabi.load()
    lib.wrnn_debug_stream_plan.restype = C.c_int
    lib.wrnn_debug_stream_plan.argtypes = [C.c_void_p] * 8 + [C.c_int32]
    cfg = cabi.WrnnCfg(512, 512, 80, 32, NCLS, cabi.MODE_RAW, {"fp16": cabi.PREC_F16, "bf16": cabi.PREC_BF16}[precision], 3)
    w = cabi.WrnnWeights()
    keep = []
    for field, key in zip(cabi.WEIGHT_FIELDS, cabi.WEIGHT_KEYS):
        a = np.ascontiguousarray(sd[key], dtype=np.float32)
        keep.append(a)
        setattr(w, field, a.ctypes.data)
    nb, nc = C.c_uint64(0), C.c_uint64(0)
    assert lib.wrnn_debug_stream_plan(C.byref(cfg), C.byref(w), None, C.byref(nb), None, C.byref(nc), None, None, only_block) == 0
    blob = np.zeros(nb.value, np.uint8)
    prog = np.zeros(nc.value, CHUNK)
    vec = np.full(4096 * 2 + 1536 * 2 + NCLS + 1, np.nan, np.float32)         # one float past b3: must stay untouched
    mine = np.zeros((4, nc.value), np.uint16)
    assert lib.wrnn_debug_stream_plan(C.byref(cfg), C.byref(w), blob.ctypes.data, C.byref(nb), prog.ctypes.data, C.byref(nc),
                                      vec.ctypes.data, mine.ctypes.data, only_block) == 0
    assert np.isnan(vec[-1]) and not np.isnan(vec[:-1]).any()
    lists = [m[m != 0xFFFF].astype(int) for m in mine]
    assert sorted(np.concatenate(lists).tolist()) == list(range(nc.value))
    for o, l in enumerate(lists):
        assert np.all(np.diff(l) > 0) and np.all(prog["owner"][l] == o)
    if only_block < 0:
        assert nc.value % 2 == 0 and np.all(prog["owner"][0::2] == prog["owner"][1::2])     # a pair travels to ONE issuing warp
    assert all(len(l) % 2 == 0 for l in lists)
    v = dict(qk=vec[:4096], vq=vec[4096:8192], b1h=vec[8192:9728], b2h=vec[9728:11264], b3=vec[11264:11264 + NCLS])
    return blob, prog, v


def tiles_of(blob, prog, precision):
    offs = np.concatenate([[0], np.cumsum(prog["size16"].astype(np.int64) * 16)])
    assert offs[-1] == blob.size
    return [decode_tile(blob[offs[i]:offs[i + 1]], int(c["nk"]) * 16, precision) for i, c in enumerate(prog)]


def scores(lg, e):
    """The kernel's score: logit - log e, in float32 (the tensor-core engines' order of the same argmax)."""
    with np.errstate(divide="ignore"):
        return (lg - np.log(e.astype(F32), dtype=F32)).astype(F32)


def best_of(sc, k0=0):
    """(score, class) of the best score of each row, ties to the lowest class."""
    k = np.argmax(sc, axis=-1)
    return np.take_along_axis(sc, k[..., None], -1)[..., 0], k + k0


def x_of(k):
    return (F32(2) * np.asarray(k).astype(F32) / F32(NCLS - 1.0) - F32(1)).astype(F32)


def raw_model_sd(seed=0):
    return helpers.state_numpy(helpers.make_model(seed, "RAW"))


# ------------------------------------------------------------------------------------------------------------------
# structure
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp16", "bf16"])
def test_raw_plan_structure(precision):
    sd = raw_model_sd()
    blob, prog, v = get_plan_raw(sd, precision)
    rnd = CT.rounder(precision)
    # the whole weight set once per step: MoL's stream with fc3 at 512 rows instead of 128
    assert blob.size == 2 * (4096 * 208 + (3 * 1536 + 2 * 512 + 512) * 512)
    assert int((prog["nk"].astype(int) * np.where(prog["b_buf2"] == B_NONE, 1, 2)).sum()) == 32 * 13 + 36 * 32 + 4 * 64 + 4 * 32 + 128
    assert np.array_equal(v["b3"], sd["fc3.bias"].astype(F32))
    f3 = prog[prog["phase"] == 4]
    assert len(f3) == 32                                            # 4 blocks x 4 owners x 2 chunks
    tiles = tiles_of(blob, prog, precision)
    W3 = rnd(sd["fc3.weight"].astype(F32))
    seen = set()
    for i in np.nonzero(prog["phase"] == 4)[0]:
        c = prog[i]
        b, o, k0 = int(c["acc"]) // 4, int(c["owner"]), int(c["k0"])
        assert int(c["acc"]) % 4 == o and 128 * o <= k0 < 128 * o + 128 and int(c["nk"]) == 4
        assert int(c["b_buf"]) == B_Y2 and int(c["b_buf2"]) == B_NONE
        assert int(c["wait_b"]) == W_Y2 | (k0 // 128) << 4            # waits for the y2 block its K range reads
        assert np.array_equal(tiles[i], W3[128 * b:128 * b + 128, k0:k0 + 64]), (b, o, k0)   # class order, no permutation
        seen.add((b, o, k0))
    assert len(seen) == 32
    # the MoL plan of the same trunk is unchanged: same chunks up to fc3, fc3 as one 30-class block
    sd_m = helpers.state_numpy(helpers.make_model(0, "MOL"))
    from test_stream_plan import get_plan
    blob_m, prog_m, v_m = get_plan(sd_m, precision)
    assert len(prog_m) == len(prog) - 24 and (prog_m["phase"] == 4).sum() == 8 and v_m["b3"].size == 128


def test_raw_cluster_rank_programs_are_the_blocks_of_the_whole_program():
    """Rank r's program is exactly the chunks of unit block r of the whole program -- fc3 block r included, so fc3 is
    split evenly over the cluster -- with the accumulators renumbered to one set per phase (fc3: set 0)."""
    sd = raw_model_sd()
    blob, prog, _ = get_plan_raw(sd)
    offs = np.concatenate([[0], np.cumsum(prog["size16"].astype(np.int64) * 16)])
    total, fc3_owner = 0, {}
    for r in range(4):
        b_r, p_r, _ = get_plan_raw(sd, only_block=r)
        o_r = np.concatenate([[0], np.cumsum(p_r["size16"].astype(np.int64) * 16)])
        sel = [i for i, c in enumerate(prog) if int(c["acc"]) // 4 == r]
        assert len(sel) == len(p_r)
        total += len(p_r)
        for o in range(4):
            a = [i for i in sel if prog["owner"][i] == o]
            b = [i for i in range(len(p_r)) if p_r["owner"][i] == o]
            assert len(a) == len(b)
            for i, j in zip(a, b):
                c, d = prog[i], p_r[j]
                for f in ("size16", "nk", "b_buf", "b_buf2", "k0", "flags", "wait_b", "phase"):
                    if f == "flags" and int(c["phase"]) == 3:
                        assert int(c[f]) & 1 == int(d[f]) & 1
                        continue
                    assert c[f] == d[f], (r, o, f, i, j)
                aset = int(c["phase"]) & 3
                assert int(d["acc"]) == 4 * aset + int(c["acc"]) % 4
                assert np.array_equal(blob[offs[i]:offs[i + 1]], b_r[o_r[j]:o_r[j + 1]])
                if int(c["phase"]) == 4:
                    fc3_owner.setdefault(int(c["acc"]) // 4, set()).add(r)
        assert (p_r["phase"] == 4).sum() == 8
    assert total == len(prog)
    assert fc3_owner == {b: {b} for b in range(4)}                  # every fc3 block belongs to exactly one rank


# ------------------------------------------------------------------------------------------------------------------
# the one-CTA program, interpreted
# ------------------------------------------------------------------------------------------------------------------
def interpret_raw(blob, prog, v, m_up, aux, expo, *, n_seg, seg_stride, steps, precision="fp16", x_force=None):
    """One CTA of the RAW stream kernel with NF = n_seg folds, in numpy (as test_stream_plan.interpret, with fc3 in
    four blocks and the running best (score, class) per fold).  Returns samples (NF, S) and logits (S, NF, 512)."""
    rnd = CT.rounder(precision)
    NF = n_seg
    L = m_up.shape[0]
    cond_z = np.concatenate([np.concatenate([m_up, aux], 1).astype(F32), np.zeros((1, CDIM), F32)])
    base = np.arange(NF) * seg_stride
    X = [np.zeros((NF, H), F32), np.zeros((NF, H), F32)]
    H2 = np.zeros((NF, H), F32)
    y2_pending = {}
    h1 = np.zeros((H, NF), F32); h2 = np.zeros((H, NF), F32)
    x = np.zeros(NF, F32)
    acc = np.zeros((16, 128, NF), F32)
    out = np.zeros((NF, steps), F32); logits = np.zeros((steps, NF, NCLS), F32)
    tiles = tiles_of(blob, prog, precision)
    for t in range(steps):
        cur = t & 1
        cond = rnd(cond_z[np.minimum(base + t, L)])
        ready = {(W_COND, 0)}
        waited = set()
        n_commit = [0] * NB
        n_arrive = [0] * NB
        xs = x.copy()
        run = (np.full(NF, -np.inf, F32), np.full(NF, NCLS, np.int64))
        fc3_done = []
        for i, c in enumerate(prog):
            blk = int(c["acc"]) // 4
            assert int(c["phase"]) == n_commit[blk]
            k0, kc = int(c["k0"]), int(c["nk"]) * 16
            if c["wait_b"]:
                wkind, wblk = int(c["wait_b"]) & 15, int(c["wait_b"]) >> 4
                key_w = (wkind, wblk) if wkind != W_COND else (wkind, 0)
                assert key_w in ready, f"chunk {i} waits for operand {key_w} not produced before it"
                waited.add(key_w)
            if int(c["b_buf"]) == B_Y2:
                assert (W_Y2, k0 // 128) in waited, f"chunk {i} reads y2 block {k0 // 128} unwaited"

            def image(buf):
                if buf == B_COND: return cond
                if buf in (B_H1PREV, B_Y1, B_Y2): return X[cur]
                if buf == B_H1NEW: return X[cur ^ 1]
                return H2
            a = int(c["acc"])
            if c["flags"] & 1:
                acc[a] = 0
            acc[a] += tiles[i] @ image(int(c["b_buf"]))[:, k0:k0 + kc].T
            if c["b_buf2"] != B_NONE:
                acc[a] += tiles[i] @ image(int(c["b_buf2"]))[:, k0:k0 + kc].T
            if c["commit"]:
                n_arrive[blk] += 1
            if not (c["commit"] and n_arrive[blk] == 4):
                continue
            b = blk
            n_arrive[b] = 0
            ph = n_commit[b]; n_commit[b] += 1
            u = slice(b * 128, b * 128 + 128)
            if ph in (0, 1):
                q0 = ph * 3 * H
                qk, vq, bh = v["qk"], v["vq"], (v["b2h"] if ph else v["b1h"])
                hs = h2 if ph else h1
                g = lambda j, arr: arr[q0 + j * H + b * 128: q0 + j * H + b * 128 + 128][:, None]
                gb = lambda j: bh[j * H + b * 128: j * H + b * 128 + 128][:, None]
                r = sig(acc[4 * b + 0] + g(0, qk) + xs[None, :] * g(0, vq) + gb(0))
                z = sig(acc[4 * b + 1] + g(1, qk) + xs[None, :] * g(1, vq) + gb(1))
                n = np.tanh(acc[4 * b + 2] + g(2, qk) + xs[None, :] * g(2, vq) + r * (acc[4 * b + 3] + gb(2))).astype(F32)
                hn = ((F32(1) - z) * n + z * hs[u]).astype(F32)
                hs[u] = hn
                (H2 if ph else X[cur ^ 1])[:, u] = rnd(hn).T
                ready.add((W_H2NEW if ph else W_H1NEW, b))
            elif ph in (2, 3):
                q0 = 6 * H + (ph - 2) * H
                y = np.maximum(((acc[4 * b] + acc[4 * b + 1]) + (acc[4 * b + 2] + acc[4 * b + 3])) + v["qk"][q0 + b * 128: q0 + b * 128 + 128][:, None]
                               + xs[None, :] * v["vq"][q0 + b * 128: q0 + b * 128 + 128][:, None], 0).astype(F32)
                if ph == 2:
                    X[cur][:, u] = rnd(y).T
                    ready.add((W_Y1, b))
                else:
                    y2_pending[b] = rnd(y).T
                    if all(nc >= 4 for nc in n_commit):
                        for bb, val in y2_pending.items():
                            X[cur][:, bb * 128: bb * 128 + 128] = val
                        y2_pending.clear()
                        for bb in range(NB): ready.add((W_Y2, bb))
            else:                                      # fc3 block b: logits, then this block's best per fold
                assert ph == 4 and b == len(fc3_done), "fc3 blocks run in class order"
                lg = (((acc[4 * b] + acc[4 * b + 1]) + (acc[4 * b + 2] + acc[4 * b + 3])) + v["b3"][u][:, None]).T.astype(F32)
                logits[t][:, u] = lg
                bs, bk = best_of(scores(lg, expo[t][:, u]), 128 * b)
                take = (bs > run[0]) | ((bs == run[0]) & (bk < run[1]))
                run = (np.where(take, bs, run[0]), np.where(take, bk, run[1]))
                fc3_done.append(b)
                if b == NB - 1:
                    x = x_of(run[1])
                    out[:, t] = x
                    if x_force is not None:
                        x = x_force[t].astype(F32)
        assert n_commit == [5, 5, 5, 5] and fc3_done == [0, 1, 2, 3]
    return out, logits


def contract_margin(lg, expo):
    """Top-two margin of the contract's argmax (log p - log e, float64) per (step, fold)."""
    with np.errstate(divide="ignore"):
        sc = lg.astype(np.float64) - np.log(expo.astype(np.float64))
    top2 = np.sort(sc, axis=-1)[..., -2:]
    return top2[..., 1] - top2[..., 0]


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
def test_raw_plan_interpreted_on_the_cpu_equals_the_engine_contract(precision):
    sd = raw_model_sd()
    w = O.hot_weights(sd)
    blob, prog, v = get_plan_raw(sd, precision)
    rs = np.random.RandomState(3)
    n_seg, seg_len, stride = 16, 32, 21
    L = (n_seg - 1) * stride + 25
    m_up, aux = rs.rand(L, 80).astype(F32), rs.randn(L, 128).astype(F32)
    expo, _ = P.raw_expo((3 << 32) | 11, 5, 40, n_seg, seg_len)
    kw = dict(n_seg=n_seg, seg_stride=stride)
    rs_x = np.random.RandomState(8)
    xf = (2.0 * rs_x.randint(0, 512, (seg_len, n_seg)) / 511.0 - 1.0).astype(F32)
    for label, x_force in (("teacher-forced", xf), ("free-running", None)):
        out, lg = interpret_raw(blob, prog, v, m_up, aux, expo, steps=seg_len, precision=precision, x_force=x_force, **kw)
        emu, lemu = CT.generate_segments(w, m_up, aux, mode="RAW", expo=expo, x_force=x_force, seg_len=seg_len,
                                         precision=precision, want_logits=True, **kw)
        err = np.abs(lg - lemu).max()
        margin = contract_margin(lemu, expo)
        got, want = np.rint((out.T + 1) * 511 / 2), np.rint((emu.T + 1) * 511 / 2)
        clear = margin > 1e-4
        if x_force is None:            # free-running: compare each fold up to its first pick that is not clear
            first = np.where((~clear).any(0), np.argmax(~clear, axis=0), seg_len)
            clear &= np.arange(seg_len)[:, None] < first[None, :]
        print(f"{precision} {label}: logits vs contract {err:.2e}; {int(clear.sum())} clear picks, "
              f"{int((got != want)[clear].sum())} differ")
        assert err <= 1e-3 and clear.mean() >= 0.9 and np.array_equal(got[clear], want[clear])


# ------------------------------------------------------------------------------------------------------------------
# cluster form: the exchange protocol, simulated
# ------------------------------------------------------------------------------------------------------------------
def simulate_cluster_raw(plans, m_up, aux, expo, *, n_seg, seg_stride, steps, precision, pick, x_force=None,
                         async_net=False, y2_to_rank0_only=False, read_before_barrier=False):
    """Four CTAs of the RAW cluster form in numpy: per rank four issuing warps and one epilogue thread, scheduled by
    `pick`.  Every 128-unit block of every image and every candidate slot carries a version tag; a read asserts the
    version it is meant to see.  Blocks are written locally and pushed to all three peers (y2 included); each rank's
    fc3 epilogue stores its (score, class) per fold into slot `rank` of every rank's table and arrives on every rank's
    candidate barrier (modelled as an mbarrier of four arrivals waited on by parity); each rank then reduces the four
    slots of its own table.  With `async_net` a push or a candidate store lands whenever the scheduler picks it.
    Negative controls: `y2_to_rank0_only` (MoL's push pattern), `read_before_barrier` (the table read without the wait)."""
    rnd = CT.rounder(precision)
    NF, R = n_seg, 4
    L = m_up.shape[0]
    cond_z = np.concatenate([np.concatenate([m_up, aux], 1).astype(F32), np.zeros((1, CDIM), F32)])
    base = np.arange(NF) * seg_stride
    progs = [p for (_, p, _) in plans]
    v = plans[0][2]
    tiles = [tiles_of(b, p, precision) for (b, p, _) in plans]
    lists = [[[i for i in range(len(p)) if p["owner"][i] == o] for o in range(4)] for p in progs]
    img = [{"X": [np.zeros((NF, H), F32) for _ in range(2)], "Hh": [np.zeros((NF, H), F32) for _ in range(2)]} for _ in range(R)]
    tag = [{(n, j, b): ("zero", -1) for n in ("X", "Hh") for j in range(2) for b in range(NB)} for _ in range(R)]
    cand = [[None] * R for _ in range(R)]                        # cand[d][r] = (step, scores, classes) in rank d's table
    bar_phase, bar_pending = [0] * R, [0] * R                    # the candidate mbarrier of each rank
    acc = [np.zeros((16, 128, NF), F32) for _ in range(R)]
    h1 = [np.zeros((H, NF), F32) for _ in range(R)]
    h2 = [np.zeros((H, NF), F32) for _ in range(R)]
    x_of_rank = [{-1: np.zeros(NF, F32)} for _ in range(R)]      # x(t) as each rank computed it
    out = np.zeros((NF, steps), F32); logits = np.zeros((steps, NF, NCLS), F32)
    pc = [[0] * 4 for _ in range(R)]
    commits = [dict() for _ in range(R)]
    drains = [[0] * 4 for _ in range(R)]
    uses = [[[0] * 4 for _ in range(4)] for _ in range(R)]
    delivered = [set() for _ in range(R)]
    epc = [0] * R
    ep_list = [[(t, ph) for t in range(steps) for ph in (0, 1, 2, 3, 4, 5)] for _ in range(R)]   # 5: the candidate reduce
    n_chunks = [[len(l) for l in lists[r]] for r in range(R)]

    def phys(buf, phase, cur):
        if buf in (B_H1PREV, B_Y1): return "X", cur
        if buf == B_H1NEW: return "X", cur ^ 1
        if buf == B_H2: return "Hh", (cur if phase <= 1 else cur ^ 1)
        return "Hh", cur

    def expected(buf, phase, t):
        if buf == B_H1PREV: return ("h1", t - 1) if t else ("zero", -1)
        if buf == B_H1NEW: return ("h1", t)
        if buf == B_H2: return (("h2", t - 1) if t else ("zero", -1)) if phase <= 1 else ("h2", t)
        if buf == B_Y1: return ("y1", t)
        return ("y2", t)

    def issuer_can_run(r, o):
        k = pc[r][o]
        if k >= steps * n_chunks[r][o]: return False
        t, j = divmod(k, n_chunks[r][o])
        c = progs[r][lists[r][o][j]]
        if c["wait_acc"] and drains[r][int(c["wait_acc"]) - 1] < uses[r][o][int(c["wait_acc"]) - 1]: return False
        if c["wait_b"]:
            kind, blk = int(c["wait_b"]) & 15, int(c["wait_b"]) >> 4
            if kind != W_COND and (kind, blk, t) not in delivered[r]: return False
        return True

    def run_chunk(r, o):
        k = pc[r][o]
        t, j = divmod(k, n_chunks[r][o])
        i = lists[r][o][j]
        c = progs[r][i]
        cur, ph = t & 1, int(c["phase"])
        if c["wait_acc"]: uses[r][o][int(c["wait_acc"]) - 1] += 1
        k0, kc = int(c["k0"]), int(c["nk"]) * 16
        a = int(c["acc"])
        if c["flags"] & 1: acc[r][a] = 0
        for buf in (int(c["b_buf"]), int(c["b_buf2"])):
            if buf == B_NONE: continue
            if buf == B_COND:
                Bm = rnd(cond_z[np.minimum(base + t, L)])
            else:
                name, jj = phys(buf, ph, cur)
                assert tag[r][(name, jj, k0 // 128)] == expected(buf, ph, t), \
                    f"rank {r} warp {o} step {t} phase {ph}: reads {name}[{jj}] block {k0 // 128} = {tag[r][(name, jj, k0 // 128)]}, wants {expected(buf, ph, t)}"
                Bm = img[r][name][jj]
            acc[r][a] += tiles[r][i] @ Bm[:, k0:k0 + kc].T
        if c["commit"]:
            commits[r][(t, ph)] = commits[r].get((t, ph), 0) + 1
        pc[r][o] += 1

    def epilogue_can_run(r):
        if epc[r] >= len(ep_list[r]): return False
        t, ph = ep_list[r][epc[r]]
        if ph == 5:                                              # mbarrier.try_wait.parity: phase t completed
            assert bar_phase[r] <= t + 1, f"rank {r}: the candidate barrier ran two phases ahead of its waiter"
            return read_before_barrier or bar_phase[r] == t + 1
        return commits[r].get((t, ph), 0) >= 4

    in_flight = []

    def land(d, name, jj, r, what, t, data):
        img[d][name][jj][:, r * 128: r * 128 + 128] = data
        tag[d][(name, jj, r)] = (what, t)
        delivered[d].add(({"h1": W_H1NEW, "h2": W_H2NEW, "y1": W_Y1, "y2": W_Y2}[what], r, t))

    def land_cand(d, r, t, bs, bk):                              # st.shared::cluster + arrive.release.cluster
        cand[d][r] = (t, bs, bk)
        bar_pending[d] += 1
        if bar_pending[d] == R:
            bar_phase[d] += 1
            bar_pending[d] = 0

    def send(fn, *args, local=False):
        if async_net and not local: in_flight.append((fn, args))
        else: fn(*args)

    def run_epilogue(r):
        t, ph = ep_list[r][epc[r]]
        cur = t & 1
        u = slice(r * 128, r * 128 + 128)
        s = ph & 3
        A = acc[r]
        xs = x_of_rank[r][t - 1]
        if ph in (0, 1):
            q0 = ph * 3 * H
            bh = v["b2h"] if ph else v["b1h"]
            hs = h2[r] if ph else h1[r]
            g = lambda j, arr: arr[q0 + j * H + r * 128: q0 + j * H + r * 128 + 128][:, None]
            gb = lambda j: bh[j * H + r * 128: j * H + r * 128 + 128][:, None]
            rr = sig(A[4 * s + 0] + g(0, v["qk"]) + xs[None, :] * g(0, v["vq"]) + gb(0))
            z = sig(A[4 * s + 1] + g(1, v["qk"]) + xs[None, :] * g(1, v["vq"]) + gb(1))
            n = np.tanh(A[4 * s + 2] + g(2, v["qk"]) + xs[None, :] * g(2, v["vq"]) + rr * (A[4 * s + 3] + gb(2))).astype(F32)
            hn = ((F32(1) - z) * n + z * hs[u]).astype(F32)
            hs[u] = hn
            name, jj, what, data = ("Hh" if ph else "X"), cur ^ 1, ("h2" if ph else "h1"), rnd(hn).T
        elif ph in (2, 3):
            q0 = 6 * H + (ph - 2) * H
            y = np.maximum(((A[4 * s] + A[4 * s + 1]) + (A[4 * s + 2] + A[4 * s + 3])) + v["qk"][q0 + r * 128: q0 + r * 128 + 128][:, None]
                           + (xs[None, :] * v["vq"][q0 + r * 128: q0 + r * 128 + 128][:, None] if ph == 2 else 0), 0).astype(F32)
            name, jj, what, data = ("X", cur, "y1", rnd(y).T) if ph == 2 else ("Hh", cur, "y2", rnd(y).T)
        if ph <= 3:
            land(r, name, jj, r, what, t, data)
            for d in range(R):
                if d != r and not (what == "y2" and y2_to_rank0_only and d != 0):
                    send(land, d, name, jj, r, what, t, data.copy())
        elif ph == 4:                                            # fc3 block r -> this rank's candidate per fold
            lg = (((A[0] + A[1]) + (A[2] + A[3])) + v["b3"][u][:, None]).T.astype(F32)
            logits[t][:, u] = lg
            bs, bk = best_of(scores(lg, expo[t][:, u]), 128 * r)
            for d in range(R):
                send(land_cand, d, r, t, bs.copy(), bk.copy(), local=(d == r))
        else:                                                    # the four candidates of this rank's table
            bs, bk = np.full(NF, -np.inf, F32), np.full(NF, NCLS, np.int64)
            for q in range(R):
                assert cand[r][q] is not None and cand[r][q][0] == t, \
                    f"rank {r} step {t}: slot {q} holds {None if cand[r][q] is None else cand[r][q][0]}, wants {t}"
                _, qs, qk = cand[r][q]
                take = (qs > bs) | ((qs == bs) & (qk < bk))
                bs, bk = np.where(take, qs, bs), np.where(take, qk, bk)
            x = x_of(bk)
            if r == 0:
                out[:, t] = x
            x_of_rank[r][t] = x_force[t].astype(F32) if x_force is not None else x
        if ph <= 4:
            drains[r][s] += 1
        epc[r] += 1

    threads = [(r, o) for r in range(R) for o in range(5)]
    n_run = 0
    while True:
        runnable = [(r, o) for (r, o) in threads if (epilogue_can_run(r) if o == 4 else issuer_can_run(r, o))]
        runnable += [(-1, k) for k in range(len(in_flight))]
        if not runnable:
            break
        r, o = pick(runnable, n_run)
        if r < 0:
            fn, args = in_flight.pop(o)
            fn(*args)
        elif o == 4: run_epilogue(r)
        else: run_chunk(r, o)
        n_run += 1
    assert all(epc[r] == len(ep_list[r]) for r in range(R)) and all(pc[r][o] == steps * n_chunks[r][o] for r in range(R) for o in range(4)), \
        "deadlock: the protocol left work undone"
    assert all(np.array_equal(x_of_rank[r][t], x_of_rank[0][t]) for r in range(R) for t in range(steps)), "ranks disagree on x"
    return out, logits


def test_raw_cluster_form_protocol_under_adversarial_schedules():
    """(a) nothing deadlocks, (b) every MMA and every candidate read sees exactly the version it is meant to, whatever
    the interleaving and however late the pushes and candidate stores land, (c) samples and logits equal the one-CTA
    interpretation bit for bit.  A single table without a per-step parity suffices: a rank stores the candidates of step
    t + 1 only once it has every y2 block of step t + 1, which each peer pushes only after reading its table of step t."""
    sd = raw_model_sd()
    plans = [get_plan_raw(sd, only_block=r) for r in range(4)]
    rs = np.random.RandomState(4)
    n_seg, stride, steps = 8, 9, 6
    Lr = (n_seg - 1) * stride + 10
    m_up, aux = rs.rand(Lr, 80).astype(F32), rs.randn(Lr, 128).astype(F32)
    expo, _ = P.raw_expo(12345, 3, 9, n_seg, steps)
    kw = dict(n_seg=n_seg, seg_stride=stride, steps=steps, precision="fp16")
    blob, prog, v = get_plan_raw(sd)
    ref_out, ref_lg = interpret_raw(blob, prog, v, m_up, aux, expo, **kw)
    rng = np.random.RandomState(0)
    schedules = {"round robin": lambda run, n: run[n % len(run)], "first runnable": lambda run, n: run[0],
                 "last runnable": lambda run, n: run[-1], "random": lambda run, n: run[rng.randint(len(run))]}
    for fav in range(4):
        schedules[f"rank {fav} eager"] = lambda run, n, fav=fav: next((x for x in run if x[0] == fav), run[0])
        schedules[f"rank {fav} lazy"] = lambda run, n, fav=fav: next((x for x in run if x[0] != fav), run[0])
        schedules[f"epilogue of rank {fav} last"] = lambda run, n, fav=fav: next((x for x in run if x != (fav, 4)), run[0])
    for name, pick in schedules.items():
        for net in (False, True):
            out, lg = simulate_cluster_raw(plans, m_up, aux, expo, pick=pick, async_net=net, **kw)
            assert np.array_equal(out, ref_out) and np.array_equal(lg, ref_lg), (name, net)
    # negative controls: MoL's y2 pattern (pushed to rank 0 only) leaves ranks 1-3 waiting for y2 forever; reading the
    # table without waiting for the candidate barrier sees another step's candidates
    with pytest.raises(AssertionError, match="deadlock"):
        simulate_cluster_raw(plans, m_up, aux, expo, pick=schedules["round robin"], y2_to_rank0_only=True, **kw)
    with pytest.raises(AssertionError, match="wants"):
        for name in ("rank 0 eager", "rank 3 lazy", "last runnable", "random"):
            simulate_cluster_raw(plans, m_up, aux, expo, pick=schedules[name], async_net=True, read_before_barrier=True, **kw)
    print(f"{len(schedules)} schedules x 2 networks: identical to the one-CTA program")
