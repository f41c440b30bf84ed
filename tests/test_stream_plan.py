"""The stream engine's packed weight stream and static step program (wavernn_b200/csrc/wrnn_stream_plan.h), checked
WITHOUT a GPU: the library exports the plan for host-resident weights (wrnn_debug_stream_plan); this test interprets it
with numpy exactly the way the kernel's issuer / epilogue warps do -- chunk by chunk, accumulator by accumulator,
the h1 ping-pong buffers, in-place h2, the barrier fields as ordering assertions -- and compares samples and logits with
the engine-arithmetic emulation oracle/contract.py (which tests/test_contract.py pins to the fp32 oracle, which
tests/test_oracle_golden.py pins to the reference's fixtures).  What remains GPU-only is the PTX (descriptors, wgmma,
mbarriers), covered by tests/test_gpu_stream.py."""
import ctypes as C

import numpy as np
import pytest

import helpers
from oracle import contract as CT
from oracle import wavernn_oracle as O
from wavernn_b200 import cabi

H, CDIM, NB = 512, 208, 4
B_COND, B_H1PREV, B_H1NEW, B_H2, B_Y1, B_Y2, B_NONE = 0, 1, 2, 3, 4, 5, 0xFF
W_NONE, W_COND, W_H1NEW, W_H2NEW, W_Y1, W_Y2 = range(6)

CHUNK = np.dtype([("size16", "<u2"), ("a_off16", "<u2"), ("acc", "u1"), ("nk", "u1"), ("b_buf", "u1"), ("b_buf2", "u1"), ("k0", "<u2"),
                  ("flags", "u1"), ("wait_b", "u1"), ("wait_acc", "u1"), ("commit", "u1"), ("owner", "u1"), ("phase", "u1")])


def get_plan(sd, precision="fp16", only_block=-1):
    lib = cabi.load()
    lib.wrnn_debug_stream_plan.restype = C.c_int
    lib.wrnn_debug_stream_plan.argtypes = [C.c_void_p] * 8 + [C.c_int32]
    cfg = cabi.WrnnCfg(512, 512, 80, 32, 30, cabi.MODE_MOL, {"fp16": cabi.PREC_F16, "bf16": cabi.PREC_BF16}[precision], 3)
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
    vec = np.zeros(4096 * 2 + 1536 * 2 + 128, np.float32)
    mine = np.zeros((4, nc.value), np.uint16)
    assert lib.wrnn_debug_stream_plan(C.byref(cfg), C.byref(w), blob.ctypes.data, C.byref(nb), prog.ctypes.data, C.byref(nc),
                                      vec.ctypes.data, mine.ctypes.data, only_block) == 0
    # the four issuing warps' lists partition the program, ascending, and agree with the owner field
    lists = [m[m != 0xFFFF].astype(int) for m in mine]
    assert sorted(np.concatenate(lists).tolist()) == list(range(nc.value))
    for o, l in enumerate(lists):
        assert np.all(np.diff(l) > 0) and np.all(prog["owner"][l] == o)
    if only_block < 0:
        assert nc.value % 2 == 0 and np.all(prog["owner"][0::2] == prog["owner"][1::2])     # a pair travels to ONE issuing warp
    assert all(len(l) % 2 == 0 for l in lists)                                                  # the issuing loop takes two records per turn
    v = dict(qk=vec[:4096], vq=vec[4096:8192], b1h=vec[8192:9728], b2h=vec[9728:11264], b3=vec[11264:])
    return blob, prog, v


def decode_tile(raw, kc, precision):
    """[128 x kc] K-major no-swizzle operand image -> dense float32 (inverse of stream::tile_index)."""
    bits = raw.view(np.uint16)
    r, k = np.meshgrid(np.arange(128), np.arange(kc), indexing="ij")
    idx = (r // 8) * (kc // 8) * 64 + (k // 8) * 64 + (r % 8) * 8 + (k % 8)
    vals = bits[idx]
    if precision == "fp16":
        return vals.view(np.float16).astype(np.float32)
    return (vals.astype(np.uint32) << 16).view(np.float32)


def sig(x):
    return (np.float32(1) / (np.float32(1) + np.exp(-x, dtype=np.float32))).astype(np.float32)


def interpret(blob, prog, v, m_up, aux, U, *, n_seg, seg_len, seg_stride, steps, precision="fp16", x_force=None):
    """One CTA of the stream kernel with NF = n_seg folds, in numpy."""
    rnd = CT.rounder(precision)
    NF = n_seg
    L = m_up.shape[0]
    cond_z = np.concatenate([np.concatenate([m_up, aux], 1).astype(np.float32), np.zeros((1, CDIM), np.float32)])
    base = np.arange(NF) * seg_stride
    X = [np.zeros((NF, H), np.float32), np.zeros((NF, H), np.float32)]       # h1 ping-pong (+ y1, then y2, in X[cur])
    H2 = np.zeros((NF, H), np.float32)
    y2_pending = {}                                                           # fc2 results held back until all fc2 MMAs are done
    h1 = np.zeros((H, NF), np.float32); h2 = np.zeros((H, NF), np.float32)   # fp32 state, [unit][fold] like the kernel's scratch
    x = np.zeros(NF, np.float32)
    acc = np.zeros((16, 128, NF), np.float32)
    out = np.zeros((NF, steps), np.float32); logits = np.zeros((steps, NF, 30), np.float32)
    nbytes = prog["size16"].astype(np.int64) * 16
    offs = np.concatenate([[0], np.cumsum(nbytes)])
    # chunks travel in pairs: the second one lands right behind the first inside the 32 KB ring slot
    assert len(prog) % 2 == 0 and np.all(prog["a_off16"][0::2] == 0) and np.all(prog["a_off16"][1::2] == prog["size16"][0::2])
    assert offs[-1] == blob.size
    tiles = [decode_tile(blob[offs[i]:offs[i + 1]], int(c["nk"]) * 16, precision) for i, c in enumerate(prog)]
    for t in range(steps):
        cur = t & 1
        cond = rnd(cond_z[np.minimum(base + t, L)])
        ready = {(W_COND, 0)}                 # staging runs ahead of the step
        waited = set()
        n_commit = [0] * NB                   # phase of each block within the step
        n_arrive = [0] * NB                   # commits of the current (phase, block): the epilogue runs after all four issuers'
        seen_owner = set()                    # (owner, phase, block) that already issued a chunk this step
        acc_drained = [True] * NB
        h2_touched = False
        xs = x.copy()
        for i, c in enumerate(prog):
            def image(buf):
                if buf == B_COND: return cond
                if buf in (B_H1PREV, B_Y1, B_Y2): return X[cur]
                if buf == B_H1NEW: return X[cur ^ 1]
                assert buf == B_H2
                return H2
            blk_of_acc = int(c["acc"]) // 4
            key = (int(c["owner"]), int(c["phase"]), blk_of_acc)
            assert int(c["phase"]) == n_commit[blk_of_acc], f"chunk {i}: phase field {c['phase']} but block {blk_of_acc} is in phase {n_commit[blk_of_acc]}"
            if key not in seen_owner:         # an issuer's first chunk of a (phase, block) must carry the accumulator-free wait
                assert int(c["wait_acc"]) == blk_of_acc + 1, f"chunk {i}: first chunk of {key} lacks wait_acc"
                assert acc_drained[blk_of_acc] or any(k[1:] == key[1:] for k in seen_owner), f"chunk {i}: block {blk_of_acc} not drained"
                seen_owner.add(key)
            else:
                assert c["wait_acc"] == 0
            k0, kc = int(c["k0"]), int(c["nk"]) * 16
            if c["wait_b"]:
                wkind, wblk = int(c["wait_b"]) & 15, int(c["wait_b"]) >> 4
                key_w = (wkind, wblk) if wkind in (W_H1NEW, W_H2NEW, W_Y1, W_Y2) else (wkind, 0)
                assert key_w in ready, f"chunk {i} waits for operand {key_w} that no epilogue of this step produces before it"
                waited.add(key_w)
            # operands are waited for per 128-unit block (h1', h2', y1) or as a whole (cond, y2); fc1's h1' read rides on its
            # h2' wait (the GRU2 epilogue of a block starts only after every h1' block has been written and waited for)
            blk_k = k0 // 128
            ph_c = int(c["phase"])
            for buf in (int(c["b_buf"]), int(c["b_buf2"])):
                if buf == B_NONE: continue
                if buf == B_COND: assert (W_COND, 0) in waited
                if buf == B_H1NEW and ph_c == 1: assert (W_H1NEW, blk_k) in waited, f"chunk {i} reads h1' block {blk_k} unwaited"
                if buf == B_H2 and (h2_touched or ph_c == 2): assert (W_H2NEW, blk_k) in waited, f"chunk {i} reads h2' block {blk_k} unwaited"
                if buf == B_Y1: assert (W_Y1, blk_k) in waited, f"chunk {i} reads y1 block {blk_k} unwaited"
                if buf == B_Y2: assert (W_Y2, blk_k) in waited, f"chunk {i} reads y2 block {blk_k} unwaited"
            a = int(c["acc"])
            if c["flags"] & 1:
                acc[a] = 0
            acc_drained[blk_of_acc] = False
            acc[a] += tiles[i] @ image(int(c["b_buf"]))[:, k0:k0 + kc].T
            if c["b_buf2"] != B_NONE:
                acc[a] += tiles[i] @ image(int(c["b_buf2"]))[:, k0:k0 + kc].T
            if c["commit"]:
                assert int(c["commit"]) - 1 == blk_of_acc
                n_arrive[blk_of_acc] += 1
            if c["commit"] and n_arrive[blk_of_acc] == 4:
                b = int(c["commit"]) - 1
                n_arrive[b] = 0
                ph = n_commit[b]; n_commit[b] += 1
                u = slice(b * 128, b * 128 + 128)
                if ph in (0, 1):                       # GRU1 / GRU2
                    q0 = ph * 3 * H
                    qk, vq, bh = v["qk"], v["vq"], (v["b2h"] if ph else v["b1h"])
                    hs = h2 if ph else h1
                    g = lambda j, arr: arr[q0 + j * H + b * 128: q0 + j * H + b * 128 + 128][:, None]
                    gb = lambda j: bh[j * H + b * 128: j * H + b * 128 + 128][:, None]
                    r = sig(acc[4 * b + 0] + g(0, qk) + xs[None, :] * g(0, vq) + gb(0))
                    z = sig(acc[4 * b + 1] + g(1, qk) + xs[None, :] * g(1, vq) + gb(1))
                    n = np.tanh(acc[4 * b + 2] + g(2, qk) + xs[None, :] * g(2, vq) + r * (acc[4 * b + 3] + gb(2))).astype(np.float32)
                    hn = ((np.float32(1) - z) * n + z * hs[u]).astype(np.float32)
                    hs[u] = hn
                    (H2 if ph else X[cur ^ 1])[:, u] = rnd(hn).T
                    if ph: h2_touched = True
                    ready.add((W_H2NEW if ph else W_H1NEW, b))
                elif ph in (2, 3):                     # fc1 / fc2
                    q0 = 6 * H + (ph - 2) * H
                    y = np.maximum(((acc[4 * b] + acc[4 * b + 1]) + (acc[4 * b + 2] + acc[4 * b + 3])) + v["qk"][q0 + b * 128: q0 + b * 128 + 128][:, None]
                                   + xs[None, :] * v["vq"][q0 + b * 128: q0 + b * 128 + 128][:, None], 0).astype(np.float32)
                    if ph == 2:
                        X[cur][:, u] = rnd(y).T
                        ready.add((W_Y1, b))
                    else:                              # y2 replaces y1 only after the LAST block's fc2 MMAs (kernel: registers)
                        y2_pending[b] = rnd(y).T
                        if n_commit == [4] * NB:
                            for bb, val in y2_pending.items():
                                X[cur][:, bb * 128: bb * 128 + 128] = val
                            y2_pending.clear()
                            for bb in range(NB): ready.add((W_Y2, bb))
                else:                                  # fc3 + sampler
                    assert b == 0 and ph == 4
                    lg = (((acc[0] + acc[1]) + (acc[2] + acc[3]))[:30] + v["b3"][:30, None]).T.astype(np.float32)
                    logits[t] = lg
                    u_t = U[t]
                    x = O.mol_sample(lg, u_t[:10 * NF].reshape(NF, 10), u_t[10 * NF:11 * NF]).astype(np.float32)
                    out[:, t] = x
                    if x_force is not None:
                        x = x_force[t].astype(np.float32)
                acc_drained[b] = True
        assert n_commit == [5, 4, 4, 4]
    return out, logits


@pytest.mark.skipif(not cabi.is_built(), reason="library not built")
@pytest.mark.parametrize("precision", ["fp16", "bf16"])
def test_stream_plan_interpreted_on_the_cpu_equals_the_engine_contract(precision):
    model = helpers.make_model(0, "MOL")
    sd = helpers.state_numpy(model)
    w = O.hot_weights(sd)
    blob, prog, v = get_plan(sd, precision)
    # structure: the whole weight set once per step, one 16-byte record per chunk
    assert blob.size == 2 * (4096 * 208 + (3 * 1536 + 2 * 512 + 128) * 512)
    assert int((prog["nk"].astype(int) * np.where(prog["b_buf2"] == B_NONE, 1, 2)).sum()) == 32 * 13 + 36 * 32 + 4 * 64 + 4 * 32 + 32
    assert set(np.unique(prog["size16"])) == {256, 1024} and prog["acc"].max() <= 15
    rs = np.random.RandomState(1)
    n_seg, seg_len, stride = 16, 40, 25
    L = (n_seg - 1) * stride + 30                                  # the last folds run past the end of the stream
    m_up, aux = rs.rand(L, 80).astype(np.float32), rs.randn(L, 128).astype(np.float32)
    U = helpers.replay_uniforms(5, seg_len, n_seg)
    kw = dict(n_seg=n_seg, seg_len=seg_len, seg_stride=stride)
    out, lg = interpret(blob, prog, v, m_up, aux, U, steps=seg_len, precision=precision, **kw)
    emu, lemu = CT.generate_segments(w, m_up, aux, uniforms=U, precision=precision, want_logits=True, **kw)
    print(precision, "plan vs contract: samples", np.abs(out - emu).max(), "logits", np.abs(lg - lemu).max())
    assert np.abs(lg - lemu).max() <= (1e-3 if precision == "fp16" else 2e-2)
    assert np.abs(out - emu).max() <= (1e-3 if precision == "fp16" else 2e-2)


@pytest.mark.skipif(not cabi.is_built(), reason="library not built")
def test_stream_plan_on_the_trained_checkpoint_teacher_forced():
    """Shipped checkpoint, real Tacotron mel, inputs forced to the reference's own samples: the interpreted plan's
    logits stay within the fp16 tolerances stated for the GPU engines (tests/test_gpu_trained.py)."""
    g = helpers.load_golden("trained_tacotron.npz")
    sd = {k: v.numpy() for k, v in helpers.pretrained_state_dict().items()}
    blob, prog, v = get_plan(sd, "fp16")
    mel = helpers.tacotron_mels()[int(g["sentence"])]
    m_up, aux = O.upsample_network(sd, O.pad_time(mel.T, 2).T, pad=2)
    U = helpers.replay_uniforms(int(g["seed"]), 12100, 4)
    steps = 120
    out, lg = interpret(blob, prog, v, m_up, aux, U, n_seg=4, seg_len=12100, seg_stride=11550, steps=steps,
                        x_force=g["raw"].T[:steps].copy())
    e = np.abs(lg - g["logits"][:steps])
    print("trained, teacher forced, interpreted plan: max", e.max(), "median", np.median(e))
    assert e.max() <= 1e-1 and np.median(e) <= 1e-3


@pytest.mark.skipif(not cabi.is_built(), reason="library not built")
def test_cluster_rank_programs_are_the_blocks_of_the_whole_program():
    """Cluster form (four CTAs split the rows of every layer): the program of rank r is exactly the chunks of unit block r
    of the whole program -- same weight tiles, same operands, K offsets, first / wait / owner / phase fields -- with the
    accumulators and their barrier ids renumbered to one set per PHASE (set = phase & 3: nothing waits for the previous
    phase's epilogue to drain); fc3 only in rank 0.  (The whole program is the one the numpy
    interpreter above checks against the engine contract.)"""
    sd = helpers.state_numpy(helpers.make_model(0, "MOL"))
    blob, prog, _ = get_plan(sd)
    nbytes = prog["size16"].astype(np.int64) * 16
    offs = np.concatenate([[0], np.cumsum(nbytes)])
    total = 0
    for r in range(4):
        b_r, p_r, _ = get_plan(sd, only_block=r)
        o_r = np.concatenate([[0], np.cumsum(p_r["size16"].astype(np.int64) * 16)])
        sel = [i for i, c in enumerate(prog) if int(c["acc"]) // 4 == r]
        assert len(sel) == len(p_r), (r, len(sel), len(p_r))
        total += len(p_r)
        # same multiset of chunks; compare per (owner, phase) in order (the interleaving across owners may differ)
        for o in range(4):
            a = [i for i in sel if prog["owner"][i] == o]
            b = [i for i in range(len(p_r)) if p_r["owner"][i] == o]
            assert len(a) == len(b)
            for i, j in zip(a, b):
                c, d = prog[i], p_r[j]
                for f in ("size16", "nk", "b_buf", "b_buf2", "k0", "flags", "wait_b", "phase"):
                    if f == "flags" and int(c["phase"]) == 3:        # the cond-release mark sits on the LAST block of the program
                        assert int(c[f]) & 1 == int(d[f]) & 1
                        continue
                    assert c[f] == d[f], (r, o, f, i, j)
                aset = int(c["phase"]) & 3
                assert int(d["acc"]) == 4 * aset + int(c["acc"]) % 4
                assert (int(c["wait_acc"]) > 0) == (int(d["wait_acc"]) > 0) and int(d["wait_acc"]) in (0, aset + 1)
                assert (int(c["commit"]) > 0) == (int(d["commit"]) > 0) and int(d["commit"]) in (0, aset + 1)
                assert np.array_equal(blob[offs[i]:offs[i + 1]], b_r[o_r[j]:o_r[j + 1]])
        assert ((p_r["flags"] & 2) > 0).sum() == 4 and (p_r["phase"] == 4).sum() == (8 if r == 0 else 0)
    assert total == len(prog)


# ------------------------------------------------------------------------------------------------------------------
# Cluster form: the exchange protocol, simulated
# ------------------------------------------------------------------------------------------------------------------
def simulate_cluster(plans, m_up, aux, U, *, n_seg, seg_stride, steps, precision, pick, x_force=None, h2_in_place=False, async_net=False):
    """Four CTAs of the cluster form in numpy: per rank four issuing warps (each walking its own chunk list) and one
    epilogue thread; a scheduler (`pick`) decides which of the 20 threads advances next, so lagging and run-ahead ranks
    are exercised.  Every rank has its own images X[0], X[1] (h1 ping-pong; y1 -> X[cur]) and Hh[0], Hh[1] (h2 ping-pong;
    y2 -> Hh[cur], rank 0 only); a finished block is written locally and pushed into the peers' images at once.  Every
    128-unit block of every image carries a version tag (what, step): a chunk asserts that each block it reads holds
    exactly the version it is meant to read -- a push that lands before a lagging peer has finished with the old content
    (or a read before the push) fails here, on the CPU.  Numerics are computed too (samples / logits).
    `h2_in_place` is the negative control: the one-CTA layout (h2 updated in place, y2 elsewhere) used in a cluster."""
    rnd = CT.rounder(precision)
    NF, R = n_seg, 4
    L = m_up.shape[0]
    cond_z = np.concatenate([np.concatenate([m_up, aux], 1).astype(np.float32), np.zeros((1, CDIM), np.float32)])
    base = np.arange(NF) * seg_stride
    progs = [p for (_, p, _) in plans]
    v = plans[0][2]
    tiles = []
    for blob, prog, _ in plans:
        offs = np.concatenate([[0], np.cumsum(prog["size16"].astype(np.int64) * 16)])
        tiles.append([decode_tile(blob[offs[i]:offs[i + 1]], int(c["nk"]) * 16, precision) for i, c in enumerate(prog)])
    lists = [[[i for i in range(len(p)) if p["owner"][i] == o] for o in range(4)] for p in progs]
    img = [{"X": [np.zeros((NF, H), np.float32) for _ in range(2)], "Hh": [np.zeros((NF, H), np.float32) for _ in range(2)]} for _ in range(R)]
    tag = [{(n, j, b): ("zero", -1) for n in ("X", "Hh") for j in range(2) for b in range(NB)} for _ in range(R)]
    acc = [np.zeros((16, 128, NF), np.float32) for _ in range(R)]
    h1 = np.zeros((H, NF), np.float32); h2 = np.zeros((H, NF), np.float32)
    x_hist = {-1: np.zeros(NF, np.float32)}                      # x(t) as broadcast by rank 0
    x_seen = [-1] * R                                            # newest sample that has landed in rank r
    out = np.zeros((NF, steps), np.float32); logits = np.zeros((steps, NF, 30), np.float32)
    # thread state
    pc = [[0] * 4 for _ in range(R)]                             # per issuer: position in its list, counted over all steps
    commits = [dict() for _ in range(R)]                         # (step, phase) -> commits so far
    drains = [[0] * 4 for _ in range(R)]                         # per accumulator set: epilogue read-outs so far
    uses = [[[0] * 4 for _ in range(4)] for _ in range(R)]       # per issuer, per set: (step, phase) openings so far
    delivered = [set() for _ in range(R)]                        # (kind, blk, step) present in rank r's images
    epc = [0] * R                                                # per epilogue thread: position in its list of (step, phase)
    ep_list = [[(t, ph) for t in range(steps) for ph in ((0, 1, 2, 3, 4) if r == 0 else (0, 1, 2, 3))] for r in range(R)]
    n_chunks = [[len(l) for l in lists[r]] for r in range(R)]

    def phys(r, buf, phase, cur):
        if buf in (B_H1PREV, B_Y1): return "X", cur
        if buf == B_H1NEW: return "X", cur ^ 1
        if buf == B_H2: return "Hh", (0 if h2_in_place else (cur if phase <= 1 else cur ^ 1))
        assert buf == B_Y2
        return "Hh", (1 if h2_in_place else cur)

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
        if c["wait_acc"]:
            s = int(c["wait_acc"]) - 1
            if drains[r][s] < uses[r][o][s]: return False        # every earlier use of the set by this warp has been read out
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
        assert a // 4 == (ph & 3)
        if c["flags"] & 1: acc[r][a] = 0
        for buf in (int(c["b_buf"]), int(c["b_buf2"])):
            if buf == B_NONE: continue
            if buf == B_COND:
                B = rnd(cond_z[np.minimum(base + t, L)])
            else:
                name, jj = phys(r, buf, ph, cur)
                assert tag[r][(name, jj, k0 // 128)] == expected(buf, ph, t), \
                    f"rank {r} warp {o} step {t} phase {ph}: reads {name}[{jj}] block {k0 // 128} = {tag[r][(name, jj, k0 // 128)]}, wants {expected(buf, ph, t)}"
                B = img[r][name][jj]
            acc[r][a] += tiles[r][i] @ B[:, k0:k0 + kc].T
        if c["commit"]:
            assert int(c["commit"]) - 1 == (ph & 3)
            commits[r][(t, ph)] = commits[r].get((t, ph), 0) + 1
        pc[r][o] += 1

    def epilogue_can_run(r):
        if epc[r] >= len(ep_list[r]): return False
        t, ph = ep_list[r][epc[r]]
        if commits[r].get((t, ph), 0) < 4: return False
        if ph == 0 and x_seen[r] < t - 1: return False           # (the kernel waits for the broadcast at the end of step t-1)
        return True

    in_flight = []                                               # bulk copies on their way: (dest, name, jj, src, what, t, data)

    def land(d, name, jj, r, what, t, data):
        img[d][name][jj][:, r * 128: r * 128 + 128] = data
        tag[d][(name, jj, r)] = (what, t)
        delivered[d].add(({"h1": W_H1NEW, "h2": W_H2NEW, "y1": W_Y1, "y2": W_Y2}[what], r, t))

    def push(r, name, jj, what, t, data, only_rank0=False):
        land(r, name, jj, r, what, t, data)                      # the local write
        for d in range(R):
            if d == r or (only_rank0 and d != 0): continue
            if async_net: in_flight.append((d, name, jj, r, what, t, data.copy()))   # lands when the scheduler says so, in any order
            else: land(d, name, jj, r, what, t, data)

    def run_epilogue(r):
        t, ph = ep_list[r][epc[r]]
        cur = t & 1
        u = slice(r * 128, r * 128 + 128)
        s = ph & 3
        A = acc[r]
        xs = x_hist[t - 1]
        if ph in (0, 1):
            q0 = ph * 3 * H
            bh = v["b2h"] if ph else v["b1h"]
            hs = h2 if ph else h1
            g = lambda j, arr: arr[q0 + j * H + r * 128: q0 + j * H + r * 128 + 128][:, None]
            gb = lambda j: bh[j * H + r * 128: j * H + r * 128 + 128][:, None]
            rr = sig(A[4 * s + 0] + g(0, v["qk"]) + xs[None, :] * g(0, v["vq"]) + gb(0))
            z = sig(A[4 * s + 1] + g(1, v["qk"]) + xs[None, :] * g(1, v["vq"]) + gb(1))
            n = np.tanh(A[4 * s + 2] + g(2, v["qk"]) + xs[None, :] * g(2, v["vq"]) + rr * (A[4 * s + 3] + gb(2))).astype(np.float32)
            hn = ((np.float32(1) - z) * n + z * hs[u]).astype(np.float32)
            hs[u] = hn
            push(r, "Hh" if ph else "X", (0 if (ph and h2_in_place) else cur ^ 1), "h2" if ph else "h1", t, rnd(hn).T)
        elif ph in (2, 3):
            q0 = 6 * H + (ph - 2) * H
            y = np.maximum(((A[4 * s] + A[4 * s + 1]) + (A[4 * s + 2] + A[4 * s + 3])) + v["qk"][q0 + r * 128: q0 + r * 128 + 128][:, None]
                           + (xs[None, :] * v["vq"][q0 + r * 128: q0 + r * 128 + 128][:, None] if ph == 2 else 0), 0).astype(np.float32)
            if ph == 2: push(r, "X", cur, "y1", t, rnd(y).T)
            else: push(r, "Hh", (1 if h2_in_place else cur), "y2", t, rnd(y).T, only_rank0=True)
        else:
            assert r == 0
            lg = (((A[0] + A[1]) + (A[2] + A[3]))[:30] + v["b3"][:30, None]).T.astype(np.float32)
            logits[t] = lg
            x = O.mol_sample(lg, U[t][:10 * NF].reshape(NF, 10), U[t][10 * NF:11 * NF]).astype(np.float32)
            out[:, t] = x
            x_hist[t] = x_force[t].astype(np.float32) if x_force is not None else x
            for d in range(R): x_seen[d] = t                     # remote stores + release.cluster arrive on every rank's BAR_X
        drains[r][s] += 1
        epc[r] += 1

    threads = [(r, o) for r in range(R) for o in range(5)]       # o == 4: the epilogue thread
    n_run = 0
    while True:
        runnable = [(r, o) for (r, o) in threads if (epilogue_can_run(r) if o == 4 else issuer_can_run(r, o))]
        runnable += [(-1, k) for k in range(len(in_flight))]     # (-1, k): the k-th copy in flight lands
        if not runnable:
            break
        r, o = pick(runnable, n_run)
        if r < 0: land(*in_flight.pop(o))
        elif o == 4: run_epilogue(r)
        else: run_chunk(r, o)
        n_run += 1
    assert all(epc[r] == len(ep_list[r]) for r in range(R)) and all(pc[r][o] == steps * n_chunks[r][o] for r in range(R) for o in range(4)), \
        "deadlock: the protocol left work undone"
    return out, logits


@pytest.mark.skipif(not cabi.is_built(), reason="library not built")
def test_cluster_form_exchange_protocol_under_adversarial_schedules():
    """The cluster form's protocol (wrnn_stream.cu, CL = 4), simulated on the CPU from the four rank programs the library
    exports: whatever the interleaving of the 4 x (4 issuing warps + epilogue) threads -- round robin, one rank running as
    far ahead as its waits allow, one rank lagging, random -- (a) nothing deadlocks, (b) every MMA reads exactly the
    version of every operand block it is meant to read (h1 / h2 ping-pong, y1 over the stale h1 image, y2 over the stale
    h2 image, blocks pushed into peers at once), (c) samples and logits equal the one-CTA interpretation bit for bit and
    the engine contract within its tolerance."""
    sd = helpers.state_numpy(helpers.make_model(0, "MOL"))
    w = O.hot_weights(sd)
    plans = [get_plan(sd, only_block=r) for r in range(4)]
    rs = np.random.RandomState(4)
    n_seg, seg_len, stride, steps = 8, 14, 9, 6
    Lr = (n_seg - 1) * stride + 10
    m_up, aux = rs.rand(Lr, 80).astype(np.float32), rs.randn(Lr, 128).astype(np.float32)
    U = helpers.replay_uniforms(7, seg_len, n_seg)
    kw = dict(n_seg=n_seg, seg_stride=stride, steps=steps, precision="fp16")
    blob, prog, v = get_plan(sd)
    ref_out, ref_lg = interpret(blob, prog, v, m_up, aux, U, seg_len=seg_len, **kw)
    emu, lemu = CT.generate_segments(w, m_up, aux, uniforms=U, precision="fp16", want_logits=True, n_seg=n_seg, seg_len=seg_len,
                                     seg_stride=stride, steps=steps)
    rng = np.random.RandomState(0)
    schedules = {"round robin": lambda run, n: run[n % len(run)], "first runnable": lambda run, n: run[0], "last runnable": lambda run, n: run[-1],
                 "random": lambda run, n: run[rng.randint(len(run))]}
    for fav in range(4):           # rank `fav` runs ahead whenever it can / lags behind whenever anything else can run
        schedules[f"rank {fav} eager"] = lambda run, n, fav=fav: next((x for x in run if x[0] == fav), run[0])
        schedules[f"rank {fav} lazy"] = lambda run, n, fav=fav: next((x for x in run if x[0] != fav), run[0])
        schedules[f"epilogue of rank {fav} last"] = lambda run, n, fav=fav: next((x for x in run if x != (fav, 4)), run[0])
    for name, pick in schedules.items():
        out, lg = simulate_cluster(plans, m_up, aux, U, pick=pick, **kw)
        assert np.array_equal(out, ref_out[:, :steps]) and np.array_equal(lg, ref_lg[:steps]), name
    # the pushes as what they are -- asynchronous copies that land some time later, in any order: as early as possible
    # ("first runnable" never picks one while a thread can run: as LATE as possible; "last runnable": at once, newest first)
    for name in ("random", "first runnable", "last runnable", "rank 2 eager", "rank 0 lazy"):
        out, lg = simulate_cluster(plans, m_up, aux, U, pick=schedules[name], async_net=True, **kw)
        assert np.array_equal(out, ref_out[:, :steps]) and np.array_equal(lg, ref_lg[:steps]), name + " (asynchronous pushes)"
    # negative control -- why h2 ping-pongs in the cluster form: updated in place (the one-CTA layout), a peer's h2' block
    # lands while a lagging rank still has GRU2 MMAs to issue on the old h2; the version check must catch that
    with pytest.raises(AssertionError, match="wants"):
        for name in ("rank 1 eager", "rank 0 lazy", "rank 3 lazy", "last runnable"):
            simulate_cluster(plans, m_up, aux, U, pick=schedules[name], h2_in_place=True, **kw)
    print(f"{len(schedules)} schedules: identical to the one-CTA program; vs contract {np.abs(ref_out[:, :steps] - emu[:, :steps]).max():.2e}")
    assert np.abs(ref_lg[:steps] - lemu[:steps]).max() <= 1e-3
