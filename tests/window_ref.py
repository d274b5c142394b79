"""The NumPy body reference (body_ref.py) carried over to engine windows: the bf16 tile GEMM in its exact regime
(enum pb2_body_e in include/pb2_engine.h), programs run one task at a time (Runner, run_program), a restatement of the
planner's read-group and fusion rules, programs whose producers and CHECK readers form read groups and fused units,
and GEMM k-chains appended to an element-wise program, for GEMM windows."""
import dataclasses

import numpy as np

import body_ref as R
from body_ref import (CHECKS, DENORM, bits_f32, fill_kinds, fma_pair_values, scattered_layout, words)
from parsec_b200 import _lib as L
from parsec_b200.bf16 import bf16_bits_to_f32, f32_to_bf16_bits
from window_harness import Layout


GEMM_EXACT_MAX = 256    # every integer of magnitude <= 256 is a bf16 value


def gemm_bf16(flows, M, N, K):
    """C (flow 2, M x N row-major bf16) += A (flow 0, M x K row-major) . B (flow 1, N x K row-major)^T, in the exact
    regime only: every operand, every partial sum and the result are integers of magnitude <= 256 (asserted, on the
    sum of magnitudes, so in any summation order).  There fp32 sums are exact and every bf16 rounding is, so the
    kernel's fused k-chains (gemm_mode 0) and its per-task units (gemm_mode 2) must both give the float64 result.
    The bytes of C after its M * N elements are left alone."""
    assert len(flows[0]) >= M * K * 2 and len(flows[1]) >= N * K * 2 and len(flows[2]) >= M * N * 2, "GEMM tiles too short"
    a = bf16_bits_to_f32(flows[0][:M * K * 2].view(np.uint16)).reshape(M, K).astype(np.float64)
    b = bf16_bits_to_f32(flows[1][:N * K * 2].view(np.uint16)).reshape(N, K).astype(np.float64)
    c = flows[2][:M * N * 2].view(np.uint16)
    c0 = bf16_bits_to_f32(c).reshape(M, N).astype(np.float64)
    with np.errstate(invalid="ignore"):
        bound = np.abs(c0) + np.abs(a) @ np.abs(b).T
        exact = all(np.array_equal(x, np.round(x)) for x in (a, b, c0))
    assert exact and bound.max(initial=0) <= GEMM_EXACT_MAX, "GEMM data outside the exact regime"
    c[:] = f32_to_bf16_bits((c0 + a @ b.T).astype(np.float32)).reshape(-1)

def run_body(body, flows, iparam=(0, 0, 0), fparam=0.0):
    """body_ref.run_body, and the bf16 tile GEMM (gemm_bf16)."""
    if body == L.BODY_GEMM_BF16:
        gemm_bf16(flows, *(int(v) for v in iparam))
        return 0
    return R.run_body(body, flows, iparam, fparam)


@dataclasses.dataclass
class Program(R.Program):
    """body_ref.Program whose DAG may be a GEMM window's and carry task priorities."""

    def dag(self, kind=0, priority=None):
        """kind: the window kind (0 HBM bodies, 1 GEMM bodies); priority: per task (queue_policy 1)."""
        d = super().dag()
        if priority is not None:
            d.tasks["priority"] = priority
        d.kind = kind
        return d


def program(p):
    """A body_ref.Program as a Program."""
    return Program(p.ntiles, list(p.tasks))


class Runner:
    """A program run task by task over copies of a layout's two images (run_program); `slot(i)` is tile i's bytes in
    the slab now."""

    def __init__(self, layout):
        self.layout = layout
        self.dev, self.host = layout.dev.copy(), layout.host.copy()
        self.valid = np.array(layout.valid, bool)
        self.version = np.zeros(len(layout.nbytes), np.uint32)
        self.result, self.seen = [], []
        self.stats = dict(bytes_h2d=0, bytes_d2h=0, stage_ins=0, body_errors=0, tasks_retired=0)

    def slot(self, i):
        return self.dev[int(self.layout.doff[i]):int(self.layout.doff[i]) + int(self.layout.nbytes[i])]

    def home(self, i):
        return self.host[int(self.layout.hoff[i]):int(self.layout.hoff[i]) + int(self.layout.nbytes[i])]

    def step(self, body, fl, ip, fp):
        st, nb = self.stats, self.layout.nbytes
        seen = np.zeros(L.MAX_FLOWS, np.uint32)
        for f, (i, acc) in enumerate(fl):
            seen[f] = self.version[i]
            if acc & L.ACCESS_READ and not self.valid[i]:
                self.slot(i)[:] = self.home(i)
                st["bytes_h2d"] += int(nb[i])
                st["stage_ins"] += 1
                self.valid[i] = True
        r = run_body(body, [self.slot(i) for i, _ in fl], ip, fp)
        if body in CHECKS:
            st["body_errors"] += r >> 32
        for i, acc in fl:
            if acc & L.ACCESS_WRITE:
                self.version[i] += 1
                self.valid[i] = True
                if acc & L.FLOW_PUSHOUT:
                    self.home(i)[:] = self.slot(i)
                    st["bytes_d2h"] += int(nb[i])
        st["tasks_retired"] += 1
        self.result.append(r)
        self.seen.append(seen)
        return r


def run_program(prog, layout):
    """The program, task by task in program order, over copies of the layout's two images.  A READ of an INVALID tile
    stages it in from its home first; a WRITE-only flow does not stage, and leaves the tile VALID; a pushout flow copies
    the whole tile home after the body.  Returns dict(dev, host, result, seen_version, state, version, stats)."""
    m = Runner(layout)
    for task in prog.tasks:
        m.step(*task)
    state = np.where(m.valid, L.TILE_VALID, L.TILE_INVALID).astype(np.int32)
    seen = np.array(m.seen, np.uint32).reshape(-1, L.MAX_FLOWS)
    return dict(dev=m.dev, host=m.host, result=np.array(m.result, np.uint64), seen_version=seen, state=state,
                version=m.version, stats=m.stats)


# ----------------------------------------------------------------------------------------------------------------------
# read groups and fused producers
# ----------------------------------------------------------------------------------------------------------------------
GROUP_MAX = 8             # PB2_GROUP_MAX (pb2_window_layout.h): members per read group
ONE_OUT = (L.BODY_FILL_I32, L.BODY_FILL_F32, L.BODY_MEMSET_U8, L.BODY_INCR_I32, L.BODY_SCALE_I32, L.BODY_ADD_IOTA_I32,
           L.BODY_IOTA_I32, L.BODY_INCR_F32)
TWO_OUT = (L.BODY_COPY, L.BODY_AXPY_F32)


def read_groups(dag, nbytes, fuse=True):
    """form_read_groups (pb2_window_plan.cpp) restated for the built-in bodies: ({leader: members} of every read group,
    {producer: members} of every fused unit).  A group is a run of 2..GROUP_MAX consecutive out-edges of one task into
    CHECK tasks that have that edge as their only input and read one tile X as their one flow; the task runs with the
    first such group as one unit when its body has a checked form writing X (flow 1 for COPY / AXPY, whose flow 0 is
    as long as X, else flow 0), no tile of it is wider than X, and it does not push X out."""
    t, n = dag.tasks, dag.ntasks
    src, dst, _ = dag.edges()
    indeg = np.minimum(np.bincount(dst, minlength=n), 2)
    indeg[dag.ready] = 2

    def reader(v):
        x = t[v]
        return (indeg[v] == 1 and x["dep_goal"] == 1 and x["body"] in CHECKS and x["nb_flows"] == 1 and x["tile"][0] >= 0
                and x["access"][0] & (L.ACCESS_RW | L.FLOW_PUSHOUT) == L.ACCESS_READ)

    def fusable(p, x):
        out = 0 if p["body"] in ONE_OUT else 1 if p["body"] in TWO_OUT else None
        if out is None or p["nb_flows"] <= out or p["tile"][out] != x or not p["access"][out] & L.ACCESS_WRITE:
            return False
        if out == 1 and nbytes[p["tile"][0]] != nbytes[x]:
            return False
        flows = [(int(p["tile"][f]), int(p["access"][f])) for f in range(p["nb_flows"]) if p["tile"][f] >= 0]
        return all(nbytes[i] <= nbytes[x] and not (i == x and a & L.ACCESS_WRITE and a & L.FLOW_PUSHOUT) for i, a in flows)

    groups, fused = {}, {}
    for u in range(n):
        out = [int(s) & ((1 << 27) - 1) for s in dag.succ[t["succ_begin"][u]:t["succ_begin"][u] + t["succ_count"][u]]]
        j, first = 0, True
        while j < len(out):
            r = j + 1
            if reader(out[j]):
                x = t[out[j]]["tile"][0]
                while r < len(out) and r - j < GROUP_MAX and reader(out[r]) and t[out[r]]["tile"][0] == x:
                    r += 1
            if r - j >= 2:
                groups[out[j]] = out[j:r]
                if fuse and first and fusable(t[u], x):
                    fused[u] = out[j:r]
                first = False
            j = r
    return groups, fused


EPISODES = ["fill_i32", "fill_f32", "memset", "incr_i32", "scale", "add_iota", "iota", "incr_f32", "copy", "axpy",
            "narrow_extra", "wide_extra", "copy_unequal", "axpy_unequal", "pushout_x", "split"]


def grouped_program(rng, layout, kinds, nepisodes):
    """A DTD program of episodes, each a producer that writes a tile X and then 2 .. GROUP_MAX + 3 CHECK readers of X
    (CHECK_I32 and CHECK_F32 on the same bits, with constants that pass and that fail, the leader's too).  kinds[i]
    says what tile i is for: "int" and "float" tiles of the main size, fma pairs "fx" / "fy" (x and y of one AXPY, of
    one size) and "ux" / "uy" (of two sizes), and "narrow" / "wide" int tiles, narrower and wider than the main size.
    The episodes cycle through EPISODES: each of the ten bodies with a checked form (WRITE or RW, on the tile's first
    use staged when the layout stages it), a FILL with a second, narrower tile (fusable) and one with a wider tile (not
    fusable), a COPY and an AXPY of unequal sizes and a FILL that pushes X out (neither fusable), and a FILL whose
    readers are split by a NOP reader.
    Returns (program, episodes): per episode dict(kind, producer, readers (task ids, the NOP's included), fusable: the
    episode's producer and the first group of its readers run as one unit under read_groups' rules (asserted to be
    what the episode was built for), members: that group, or the first group when there is no fused unit)."""
    nt = len(kinds)
    of = lambda k: [i for i in range(nt) if kinds[i] == k]
    pools = {k: of(k) for k in ("int", "float", "fx", "ux", "narrow", "wide")}
    turn = {k: 0 for k in pools}

    def pick(k):
        i = pools[k][turn[k] % len(pools[k])]
        turn[k] += 1
        return i

    prog = Program(nt)
    m = Runner(layout)

    def task(body, flows, ip=(0, 0, 0), fp=0.0):
        ip = tuple(int(v) for v in ip)
        m.step(body, flows, ip, fp)
        return prog.task(body, flows, ip, fp)

    def filler():
        return L.ACCESS_WRITE if rng.random() < 0.5 else L.ACCESS_RW

    episodes = []
    for e in range(nepisodes):
        kind = EPISODES[e % len(EPISODES)]
        want = kind not in ("wide_extra", "copy_unequal", "axpy_unequal", "pushout_x")
        x = pick("float" if kind in ("incr_f32",) else "int")
        k = int(rng.integers(-3, 4))
        if kind in ("fill_i32", "narrow_extra", "wide_extra", "pushout_x", "split"):
            flows = [(x, filler() | (L.FLOW_PUSHOUT if kind == "pushout_x" else 0))]
            if kind in ("narrow_extra", "wide_extra"):
                flows.append((pick("narrow" if kind == "narrow_extra" else "wide"), L.ACCESS_READ))
            p = task(L.BODY_FILL_I32, flows, (int(rng.integers(-(1 << 31), 1 << 31)) if e % 3 else k, 0, 0))
        elif kind == "fill_f32":
            if e % 2:
                x = pick("float")
            p = task(L.BODY_FILL_F32, [(x, filler())], fp=float(rng.choice([1.5, -2.25, 0.0, -0.0, float(bits_f32(DENORM))])))
        elif kind == "memset":
            p = task(L.BODY_MEMSET_U8, [(x, filler())], (int(rng.choice([0, 1, 0xA5, 0x3C])), 0, 0))
        elif kind == "iota":
            p = task(L.BODY_IOTA_I32, [(x, filler())])
        elif kind in ("incr_i32", "scale", "add_iota"):
            body = {"incr_i32": L.BODY_INCR_I32, "scale": L.BODY_SCALE_I32, "add_iota": L.BODY_ADD_IOTA_I32}[kind]
            p = task(body, [(x, L.ACCESS_RW)], (k, 0, 0))
        elif kind == "incr_f32":
            p = task(L.BODY_INCR_F32, [(x, L.ACCESS_RW)], fp=float(rng.choice([1.5, -2.25, 0.0625, -0.0])))
        elif kind in ("copy", "copy_unequal"):
            a = pick("narrow") if kind == "copy_unequal" else pick("int")
            if a == x:
                a = pick("int")
            p = task(L.BODY_COPY, [(a, L.ACCESS_READ), (x, filler())])
        else:                                       # axpy, axpy_unequal: the pair's one AXPY
            a = pick("ux" if kind == "axpy_unequal" else "fx")
            x = a + 1
            p = task(L.BODY_AXPY_F32, [(a, L.ACCESS_READ), (x, L.ACCESS_RW)], fp=float(fma_pair_values(rng, 1)[2]))
        first = int(words(m.slot(x))[0]) if m.layout.nbytes[x] >= 4 else 0
        nread = int(rng.integers(4 if kind == "split" else 2, GROUP_MAX + 4))
        split = int(rng.integers(1, nread)) if kind == "split" else -1     # the NOP goes before reader `split`
        readers = []
        for r in range(nread):
            if r == split:
                readers.append(task(L.BODY_NOP, [(x, L.ACCESS_READ)]))
            passing = rng.random() < (0.3 if r == 0 else 0.5)
            c = first if passing else int(rng.choice([first ^ 1, first + 7, 0, 3])) & 0xFFFFFFFF
            f = bits_f32(c)
            if rng.random() < 0.5 and not np.isnan(f):
                readers.append(task(L.BODY_CHECK_F32, [(x, L.ACCESS_READ)], fp=f))
            else:
                readers.append(task(L.BODY_CHECK_I32, [(x, L.ACCESS_READ)], (c - (1 << 32) if c >= 1 << 31 else c, 0, 0)))
        episodes.append(dict(kind=kind, producer=p, readers=readers, want=want))
    groups, fused = read_groups(prog.dag(), layout.nbytes)
    for ep in episodes:
        p = ep.pop("want")
        ep["fusable"] = ep["producer"] in fused
        assert ep["fusable"] == p, ("episode built for another rule", ep)
        heads = [r for r in ep["readers"] if r in groups]
        ep["members"] = fused[ep["producer"]] if ep["fusable"] else groups[heads[0]] if heads else []
    return prog, episodes


def grouped_case(seed, size, staged, nepisodes=32):
    """A grouped program over tiles of `size` bytes (and narrower and wider ones) on a scattered layout whose tiles all
    start INVALID (staged) or VALID: (program, layout, episodes)."""
    rng = np.random.default_rng(seed)
    kinds = ["int"] * 10 + ["float"] * 3 + ["fx", "fy"] * 2 + ["ux", "uy", "narrow", "narrow", "wide", "wide"]
    narrow, wide = max(size // 2 - 3, 1), size + 20
    sizes = [{"narrow": narrow, "wide": wide, "uy": size - 4 if size >= 8 else wide}.get(k, size) for k in kinds]
    layout = scattered_layout(rng, sizes, np.full(len(sizes), not staged))
    fill_kinds(rng, layout, ["float" if k == "float" else "fx" if k in ("fx", "ux") else "int" for k in kinds])
    prog, episodes = grouped_program(rng, layout, kinds, nepisodes)
    return prog, layout, episodes


# ----------------------------------------------------------------------------------------------------------------------
# GEMM k-chains beside element-wise programs (GEMM windows)
# ----------------------------------------------------------------------------------------------------------------------
GEMM_CHAINS = ((7, 264, 72, 3), (64, 776, 8, 2))      # M, N, K, tasks in the chain


def with_gemm_chains(rng, prog, layout, copy_to, chains=GEMM_CHAINS):
    """prog and layout with exact-regime GEMM k-chains appended, each on tiles of its own: operands with entries in
    {-1, 0, 1} (about six nonzero products per dot product) and C with integers in [-3, 3], every tile followed by some
    padding, some staged and some resident, homes 16-, 4- and 1-byte aligned in turn; the first chain's last task
    pushes C out.  After each chain three CHECKs read its C (a read group, which a GEMM never fuses with), and after the
    last one a COPY takes the first chain's C into int tile copy_to, which two CHECKs then read.  Returns (program,
    layout)."""
    nb, doff, hoff, valid = list(layout.nbytes), list(layout.doff), list(layout.hoff), list(layout.valid)
    d, h = len(layout.dev), len(layout.host)
    data = []

    def tile(values, pad, resident):
        nonlocal d, h
        b = f32_to_bf16_bits(np.asarray(values, np.float32)).reshape(-1).view(np.uint8)
        n = len(b) + pad
        h = (h + 8 + 15) // 16 * 16 + (0, 4, 3)[len(nb) % 3]
        doff.append(d), hoff.append(h), nb.append(n), valid.append(resident)
        data.append(b)
        d = (d + n + 48 + 127) // 128 * 128 + 16
        h += n
        return len(nb) - 1

    out = Program(prog.ntiles, list(prog.tasks))
    cs = []
    for c, (M, N, K, length) in enumerate(chains):
        p = min(0.5, float(np.sqrt(6.0 / K)))
        tern = lambda shape: np.where(rng.random(shape) < p, np.where(rng.random(shape) < 0.5, -1.0, 1.0), 0.0)
        ops = [(tile(tern((M, K)), 34, j % 2 == 0), tile(tern((N, K)), 130, j % 3 == 1)) for j in range(length)]
        C = tile(rng.integers(-3, 4, (M, N)), 6, c == 0)
        cs.append(C)
        for j, (A, B) in enumerate(ops):
            push = L.FLOW_PUSHOUT if c == 0 and j == length - 1 else 0
            out.task(L.BODY_GEMM_BF16, [(A, L.ACCESS_READ), (B, L.ACCESS_READ), (C, L.ACCESS_RW | push)], (M, N, K))
        for k in (0x3F803F80, 0, 0x3F803F80):        # two bf16 1.0; 0
            out.task(L.BODY_CHECK_I32, [(C, L.ACCESS_READ)], (k, 0, 0))
        out.task(L.BODY_CHECK_F32, [(C, L.ACCESS_READ)], fparam=bits_f32(0x3F803F80))
    out.task(L.BODY_COPY, [(cs[0], L.ACCESS_READ), (copy_to, L.ACCESS_WRITE)])
    out.task(L.BODY_CHECK_I32, [(copy_to, L.ACCESS_READ)])
    out.task(L.BODY_CHECK_F32, [(copy_to, L.ACCESS_READ)], fparam=bits_f32(0x3F803F80))
    dev = np.concatenate([layout.dev, np.full(d - len(layout.dev), 0xA5, np.uint8)])
    host = np.concatenate([layout.host, np.full(h + 16 - len(layout.host), 0x3C, np.uint8)])
    first = len(layout.nbytes)
    for j, b in enumerate(data):
        i = first + j
        n = int(nb[i])
        host[hoff[i]:hoff[i] + n] = rng.integers(0, 4, n, dtype=np.uint8)
        host[hoff[i]:hoff[i] + len(b)] = b
        if valid[i]:
            dev[doff[i]:doff[i] + n] = rng.integers(0, 4, n, dtype=np.uint8)
            dev[doff[i]:doff[i] + len(b)] = b
    out.ntiles = len(nb)
    return out, Layout(np.array(doff, np.int64), np.array(hoff, np.int64), np.array(nb, np.int64), np.array(valid, bool),
                       dev, host)

