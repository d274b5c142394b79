"""Windows that mix tile GEMMs with HBM bodies on the H100: the stand-alone runtime runs the mixed DTD pool in one
launch, the GEMM kernel runs random mixed DAGs exactly as the sequential oracle does (DESIGN §6), and wide HBM bodies
of a GEMM window are cut into byte-slice parts whose CHECK results add up exactly."""
import dataclasses

import numpy as np
import pytest

from oracle import orc
from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
from parsec_b200.bf16 import bf16_bits_to_f32, f32_to_bf16_bits
from parsec_b200.engine import Engine
from priority_order import LANES, priority_order, replay
import mixed_pool as P
from window_harness import Layout, assert_like_oracle, placed, run_oracle

pytestmark = pytest.mark.gpu

PART = 256 * 1024          # the engine's default part_bytes


# ----------------------------------------------------------------------------------------------------------------------
# 1. the mixed DTD pool through the stand-alone runtime
# ----------------------------------------------------------------------------------------------------------------------
def test_mixed_pool_runs_in_one_launch():
    NT, T = 2, 1024                                   # C tiles of 2 MiB: FILL, CHECK and AXPY run as 8 parts each
    data = P.Data(NT, T, seed=1)
    init = data.host.copy()
    # the oracle runs the window the runtime builds for the same pool, on a copy of the same data
    odata = P.Data(NT, T, seed=1)
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        tp, oids = P.insert(ctx, odata)
        win = ctx.export_window(tp, ctx.devices[0])
    spec = win["tiles"].copy()
    spec["src_ptr"] = spec["src_ptr"] - np.uint64(odata.host.ctypes.data)
    ohost = odata.host.copy()
    o = orc.run_window(win["tasks"], win["succ"], spec, win["ready"], ohost)
    assert o["rc"] == 0
    n = P.ntasks(NT)
    oseen, ores = np.zeros((n, 4), np.uint32), np.zeros(n, np.uint64)
    oseen[win["task_ids"]], ores[win["task_ids"]] = o["seen_version"], o["result"]

    # tiles come in through the kernels' stage-in (the parts of the AXPYs pull X slice by slice), not the copy engine
    with R.Context(cuda_devices=(0,), mca={"device_engine_dma_prefetch_min_bytes": 0}) as ctx:
        tp, ids = P.insert(ctx, data)
        ctx.wait()
        st = ctx.stats(ctx.devices[0])
        info = ctx.task_info(tp)
        order, dev = ctx.trace(tp)
        assert ctx.l.pb2_device_memory_release(ctx.devices[0]) == 0
    assert ids == oids
    assert sorted(order.tolist()) == list(range(n)) and np.all(dev == 2)
    assert st["windows_launched"] == 1 and st["executed_tasks"] == n
    assert st["tasks_released_on_device"] == n - P.nready(NT)
    assert np.array_equal(info["seen_version"], oseen)

    # integer tiles: bit for bit the oracle's, and the known answer Y = Y0 + 2 X0
    got = data.view("Y")
    assert np.array_equal(got, ohost[P.NAMES.index("Y") * data.mat_bytes:][:data.mat_bytes])
    x0 = init[P.NAMES.index("X") * data.mat_bytes:][:data.mat_bytes].view(np.float32)
    y0 = init[P.NAMES.index("Y") * data.mat_bytes:][:data.mat_bytes].view(np.float32)
    assert np.array_equal(got.view(np.float32), y0 + np.float32(P.ALPHA) * x0)
    for name in ("A", "B", "X"):
        assert np.array_equal(data.view(name), init[P.NAMES.index(name) * data.mat_bytes:][:data.mat_bytes]), name

    # GEMM values: within one bf16 ulp of the largest magnitude along the k-chain (DESIGN §7)
    for i in range(NT):
        for j in range(NT):
            acc = np.ones((T, T), np.float64)
            big = np.abs(acc)
            for k in range(NT):
                a = bf16_bits_to_f32(data.tile("A", i, k).view(np.uint16)).reshape(T, T).astype(np.float64)
                b = bf16_bits_to_f32(data.tile("B", k, j).view(np.uint16)).reshape(T, T).astype(np.float64)
                acc = acc + a @ b.T
                big = np.maximum(big, np.abs(acc))
            c = data.tile("C", i, j)
            gc = bf16_bits_to_f32(c.view(np.uint16)).reshape(T, T).astype(np.float64)
            assert np.all(np.abs(gc - acc) <= 2.0 ** -7 * big), (i, j, float(np.max(np.abs(gc - acc) / big)))
            # the CHECK after the chain saw the chain's output: every word that is not two bf16 1.0 counts
            words = c.view(np.uint32)
            want_r = (int(np.count_nonzero(words != P.ONES)) << 32) | int(words[0])
            assert int(info["result"][ids[("check", i, j)]]) == want_r, (i, j)


# ----------------------------------------------------------------------------------------------------------------------
# 2. random mixed DAGs on the GEMM kernel against the oracle
# ----------------------------------------------------------------------------------------------------------------------
M, N, K = 256, 256, 128
OP = {L.ACCESS_READ: orc.DTD_INPUT, L.ACCESS_WRITE: orc.DTD_OUTPUT, L.ACCESS_RW: orc.DTD_INOUT}


class MixedDag:
    """A random DTD program over wide integer tiles (ragged byte sizes), float tiles, and the A / B / C tiles of
    GEMM k-chains whose outputs are copied and checked by HBM bodies.  Every value stays an exact integer: GEMM
    operands in {-1, 0, 1}, C bounded by 256 (checked), AXPY with alpha = +-1 on small integers."""

    def __init__(self, seed, ntasks=160, nprio=1):
        rng = np.random.default_rng(seed)
        kinds, sizes = [], []
        for _ in range(6):
            kinds.append("int"); sizes.append(4 * int(rng.integers(60_000, 300_000)))
        for _ in range(3):
            kinds.append("flt"); sizes.append(4 * int(rng.integers(60_000, 200_000)))
        for what, nb in (("A", M * K * 2), ("B", N * K * 2), ("B", N * K * 2), ("A", M * K * 2), ("C", M * N * 2),
                         ("C", M * N * 2), ("C", M * N * 2)):
            kinds.append(what); sizes.append(nb)
        self.kinds, self.bytes = kinds, np.array(sizes, np.int64)
        of = lambda k: [i for i, x in enumerate(kinds) if x == k]
        ints, flts, As, Bs, Cs = of("int"), of("flt"), of("A"), of("B"), of("C")
        self.init = []
        for k, nb in zip(kinds, sizes):
            if k == "int":
                self.init.append(rng.integers(-50, 50, nb // 4).astype(np.int32).view(np.uint8))
            elif k == "flt":
                self.init.append(rng.integers(-50, 50, nb // 4).astype(np.float32).view(np.uint8))
            elif k == "C":
                self.init.append(f32_to_bf16_bits(rng.integers(-2, 3, nb // 2).astype(np.float32)).view(np.uint8))
            else:
                v = np.where(rng.random(nb // 2) < 0.04, np.where(rng.random(nb // 2) < 0.5, -1.0, 1.0), 0.0)
                self.init.append(f32_to_bf16_bits(v.astype(np.float32)).view(np.uint8))
        rows, naxpy = [], 0
        for _ in range(ntasks):
            u = rng.random()
            pick = lambda xs: int(rng.choice(xs))
            if u < 0.30:
                rows.append((L.BODY_GEMM_BF16, [(pick(As), L.ACCESS_READ), (pick(Bs), L.ACCESS_READ), (pick(Cs), L.ACCESS_RW)], (M, N, K), 0.0))
            elif u < 0.38:
                t = pick(ints + Cs)
                v = int(rng.integers(-9, 9)) if kinds[t] == "int" else int(rng.choice([0, P.ONES]))
                rows.append((L.BODY_FILL_I32, [(t, L.ACCESS_WRITE)], (v, 0, 0), 0.0))
            elif u < 0.46:
                rows.append((L.BODY_SCALE_I32, [(pick(ints), L.ACCESS_RW)], (int(rng.integers(-2, 4)), 0, 0), 0.0))
            elif u < 0.54:
                rows.append((L.BODY_INCR_I32, [(pick(ints), L.ACCESS_RW)], (int(rng.integers(-5, 6)), 0, 0), 0.0))
            elif u < 0.66:
                src = pick(ints + Cs)
                dst = pick([x for x in (ints if kinds[src] == "int" or rng.random() < 0.5 else Cs) if x != src])
                if kinds[dst] == "C" and kinds[src] != "C":
                    dst = pick(ints)
                rows.append((L.BODY_COPY, [(src, L.ACCESS_READ), (dst, L.ACCESS_RW)], (0, 0, 0), 0.0))
            elif u < 0.74 and naxpy < 12:
                x, y = rng.choice(flts, 2, replace=False)
                naxpy += 1
                rows.append((L.BODY_AXPY_F32, [(int(x), L.ACCESS_READ), (int(y), L.ACCESS_RW)], (0, 0, 0), float(rng.choice([1.0, -1.0]))))
            elif u < 0.82:
                # bodies that use the part's element offset (BodyArgs::elem0)
                t = pick(ints)
                which = int(rng.integers(0, 3))
                if which == 0:
                    rows.append((L.BODY_IOTA_I32, [(t, L.ACCESS_WRITE)], (0, 0, 0), 0.0))
                elif which == 1:
                    rows.append((L.BODY_ADD_IOTA_I32, [(t, L.ACCESS_RW)], (0, 0, 0), 0.0))
                else:
                    at = int(rng.integers(0, sizes[t] // 4))
                    rows.append((L.BODY_ADD_AT_I32, [(t, L.ACCESS_RW)], (at, int(rng.integers(1, 1000)), 0), 0.0))
            else:
                t = pick(ints + flts + Cs)
                k = int(rng.choice([0, P.ONES, int(rng.integers(-9, 9))]))
                rows.append((L.BODY_CHECK_I32, [(t, L.ACCESS_READ)], (k, 0, 0), 0.0))
        # pushout on a fifth of the written flows
        rows = [(b, [(t, a | (L.FLOW_PUSHOUT if (a & L.ACCESS_WRITE) and rng.random() < 0.2 else 0)) for t, a in fl], ip, fp)
                for b, fl, ip, fp in rows]
        n = len(rows)
        t = np.zeros(n, L.TASK_DTYPE)
        t["tile"][:] = -1
        ft, fo = np.full((n, 4), -1, np.int32), np.zeros((n, 4), np.int32)
        for i, (body, fl, ip, fp) in enumerate(rows):
            t["body"][i], t["nb_flows"][i], t["iparam"][i], t["fparam"][i] = body, len(fl), ip, fp
            t["priority"][i] = int(rng.integers(0, nprio))
            for f, (tile, acc) in enumerate(fl):
                t["tile"][i, f], t["access"][i, f] = tile, acc
                ft[i, f], fo[i, f] = tile, OP[acc & L.ACCESS_RW]
        src, dst, flow, dep = orc.dtd_build(t["nb_flows"].astype(np.int32), ft, fo, len(kinds))
        begin, count, succ = dags._csr_from_edges(n, src, dst, flow)
        t["succ_begin"], t["succ_count"], t["dep_goal"] = begin, count, dep
        self.dag = dags.Dag(t, succ, np.nonzero(dep == 0)[0].astype(np.int32), ntiles=len(kinds), tile_bytes=0, kind=1)
        # exact regime: no C element can leave [-256, 256] whatever the order of the GEMMs (bf16 then rounds nothing)
        absprod = {}
        bound = 2
        for i, (body, fl, _, _) in enumerate(rows):
            if body == L.BODY_GEMM_BF16:
                a, b = fl[0][0], fl[1][0]
                if (a, b) not in absprod:
                    av = np.abs(bf16_bits_to_f32(self.init[a].view(np.uint16)).reshape(M, K))
                    bv = np.abs(bf16_bits_to_f32(self.init[b].view(np.uint16)).reshape(N, K))
                    absprod[(a, b)] = float((av @ bv.T).max())
                bound += absprod[(a, b)]
        assert bound <= 256, f"seed {seed}: GEMM data outside the exact regime ({bound})"
        # slab (16-byte aligned slots, gaps between them) and host image; `valid` tiles start resident.  Host copies
        # sit back to back from byte 4 on: most are only 4-byte aligned, as the tiles of a collection of odd-sized
        # tiles are, so pushout and stage-in take the narrow copy loops
        self.valid = rng.random(len(kinds)) < 0.4
        self.doff, self.hoff = np.zeros(len(kinds), np.int64), np.zeros(len(kinds), np.int64)
        d, h = 0, 4
        for i, nb in enumerate(sizes):
            self.doff[i], self.hoff[i] = d, h
            d += (nb + 64 + 127) // 128 * 128
            h += nb
        dev = np.full(d, 0xAB, np.uint8)
        host = np.zeros(h, np.uint8)
        for i, x in enumerate(self.init):
            host[self.hoff[i]:self.hoff[i] + len(x)] = x
            if self.valid[i]:
                dev[self.doff[i]:self.doff[i] + len(x)] = x
        self.layout = Layout(self.doff, self.hoff, self.bytes, self.valid, dev, host)

    def nparts(self, part_bytes):
        """Ring entries per task as build_gemm2_units (pb2_window_plan.cpp) cuts a GEMM window's HBM units (GEMM tasks: 0, not checked)."""
        t, out = self.dag.tasks, np.zeros(self.dag.ntasks, np.int64)
        pb = PART if part_bytes == 0 else part_bytes
        for i in range(len(t)):
            if t["body"][i] == L.BODY_GEMM_BF16:
                continue
            widest = max(int(self.bytes[t["tile"][i, f]]) for f in range(t["nb_flows"][i]))
            out[i] = min(-(-widest // pb), 32) if pb > 0 and t["body"][i] != L.BODY_NOP else 1
        return out



def run_with_parts(eng, md, layout):
    """A run of md's window over layout, with res["parts"]: the ring entries of every task."""
    with placed(eng, layout) as p:
        w = eng.window(1, md.dag.tasks, md.dag.succ, p.tiles, md.dag.ready)
        try:
            st, res = w.run(), w.results()
            res["parts"] = (w.task_entries().view(np.uint32) >> np.uint32(27)).astype(np.int64) + 1
        finally:
            w.close()
    return p.run(st, res, images=(p.dev, p.host))


def assert_cut_into_parts(md, res, part_bytes):
    """The window's HBM units have the part counts of the rule (pb2_window_task_entries: parts - 1 in the part field).
    A unit retires only when all its parts have run (parts_left), so a window that retired every task ran them all."""
    want = md.nparts(part_bytes)
    hbm = md.dag.tasks["body"] != L.BODY_GEMM_BF16
    assert np.array_equal(res["parts"][hbm], want[hbm])
    assert np.count_nonzero(want > 1) > 10


@pytest.mark.parametrize("seed", [21, 22, 23])
@pytest.mark.parametrize("engine_kw", [dict(), dict(part_bytes=65536), dict(gemm_mode=2, part_bytes=16384)],
                         ids=["default", "parts64k", "per_task_units_parts16k"])
def test_random_mixed_dag_all_workers(seed, engine_kw):
    md = MixedDag(seed)
    with Engine(0, timeout_ms=8000, **engine_kw) as e:
        got = run_with_parts(e, md, md.layout)
    assert_like_oracle(got, run_oracle(md.dag, md.layout), md.dag)
    assert_cut_into_parts(md, got.res, engine_kw.get("part_bytes", 0))


@pytest.mark.parametrize("seed", [31, 32])
def test_random_mixed_dag_one_worker_retires_in_fifo_order(seed):
    """(5): with one worker and every task its own unit, the retire order is the oracle's FIFO order; the wide HBM
    bodies run as parts (a unit's parts are consecutive ring entries)."""
    md = MixedDag(seed, ntasks=120)
    want = run_oracle(md.dag, md.layout)
    with Engine(0, max_workers=1, gemm_mode=2, timeout_ms=8000) as e:
        got = run_with_parts(e, md, md.layout)
    assert_like_oracle(got, want, md.dag)
    assert np.array_equal(got.res["retire_order"], want.res["retire_order"])
    assert_cut_into_parts(md, got.res, 0)


def test_random_mixed_dag_one_worker_priority_lanes():
    """queue_policy 1, one worker: the order of tests/priority_order.py (GEMM windows form no read groups), and the
    oracle's bytes when it runs the tasks in that order."""
    md = MixedDag(41, ntasks=120, nprio=40)
    assert len(np.unique(md.dag.tasks["priority"])) > LANES
    order = priority_order(md.dag, LANES)
    staged = dataclasses.replace(md.layout, valid=np.zeros(md.dag.ntiles, bool))
    ohost = staged.host.copy()
    ref = replay(md.dag, order, staged.offsets(), ohost)
    with Engine(0, max_workers=1, gemm_mode=2, queue_policy=1, part_bytes=65536, timeout_ms=8000) as e:
        st, res, dev, host, _, _ = run_with_parts(e, md, staged)
    assert st["tasks_retired"] == md.dag.ntasks
    assert_cut_into_parts(md, res, 65536)
    assert np.array_equal(res["retire_order"], order)
    assert all(v == 0 for v in dags.check_execution(md.dag, res).values())
    assert np.array_equal(res["seen_version"], ref["seen_version"])
    assert np.array_equal(res["result"], ref["result"])
    assert np.array_equal(res["tiles"]["version"], ref["tiles"]["version"])
    for i in range(md.dag.ntiles):
        a = staged.tile_bytes(dev, i)
        assert np.array_equal(a, ref["device"][i][:len(a)]), i
    assert np.array_equal(host, ohost)


# ----------------------------------------------------------------------------------------------------------------------
# 3. wide CHECK parts add their mismatch counts exactly
# ----------------------------------------------------------------------------------------------------------------------
def part_cut(nbytes, part_bytes):
    """(nparts, bytes per part) of a one-flow task, by the rule of build_gemm2_units (pb2_window_plan.cpp) / run_task_part."""
    np_ = min(-(-nbytes // part_bytes), 32) if part_bytes > 0 else 1
    return np_, ((nbytes // np_) + 15) & ~15


@pytest.mark.parametrize("part_bytes", [0, 65536, -1], ids=["default", "64k", "one_part"])
def test_wide_check_parts_add_up(part_bytes):
    K32 = 0x01234567
    FK = np.float32(3.5)
    sizes = [2 * 1024 * 1024 + 12, 1 << 20, 3 * 1024 * 1024 + 4, 8 * 1024 * 1024 + 20, 4096 + 8]
    pb = PART if part_bytes == 0 else part_bytes
    tiles, counts = [], []
    rng = np.random.default_rng(5)
    for ti, nb in enumerate(sizes):
        f32 = ti == 2
        words = np.full(nb // 4, FK.view(np.uint32) if f32 else K32, np.uint32)
        nparts, per = part_cut(nb, pb)
        bad = set()
        if ti != 1:                                           # tile 1: no mismatch at all
            for p in range(nparts):                           # known mismatches in known slices: p + 1 in slice p
                lo, hi = p * per // 4, min((p + 1) * per, nb) // 4
                bad |= set(int(x) for x in rng.choice(np.arange(lo, hi), min(p + 1, hi - lo), replace=False))
                bad |= {lo, hi - 1}                               # both ends of every slice
            bad.add(len(words) - 1)                            # the ragged tail's last element
        if ti == 3:
            bad |= set(range(1000, 3000))                      # a dense run inside slice 0
        for x in bad:
            words[x] ^= 0x00010000
        tiles.append(words.view(np.uint8))
        counts.append(len(bad))
    # one small GEMM makes it a GEMM window; its C is a tile of its own
    ab = f32_to_bf16_bits(np.ones(128 * 128, np.float32)).view(np.uint8)
    tiles += [ab, ab.copy(), np.zeros(128 * 128 * 2, np.uint8)]
    nt = len(tiles)
    t = np.zeros(len(sizes) + 1, L.TASK_DTYPE)
    t["tile"][:] = -1
    for i in range(len(sizes)):
        t["body"][i], t["nb_flows"][i] = (L.BODY_CHECK_F32 if i == 2 else L.BODY_CHECK_I32), 1
        t["tile"][i, 0], t["access"][i, 0] = i, L.ACCESS_READ
        t["iparam"][i, 0], t["fparam"][i] = K32, FK
    g = len(sizes)
    t["body"][g], t["nb_flows"][g], t["iparam"][g] = L.BODY_GEMM_BF16, 3, (128, 128, 128)
    t["tile"][g, :3], t["access"][g, :3] = (nt - 3, nt - 2, nt - 1), (L.ACCESS_READ, L.ACCESS_READ, L.ACCESS_RW)
    off = np.zeros(nt, np.int64)
    for i in range(1, nt):
        off[i] = off[i - 1] + (len(tiles[i - 1]) + 127) // 128 * 128
    image = np.zeros(int(off[-1]) + len(tiles[-1]), np.uint8)
    for i, x in enumerate(tiles):
        image[off[i]:off[i] + len(x)] = x
    with Engine(0, part_bytes=part_bytes, timeout_ms=8000) as e:
        slab = e.malloc(len(image))
        e.h2d(slab, image)
        tl = np.zeros(nt, L.TILE_DTYPE)
        tl["dev_ptr"] = slab + off.astype(np.uint64)
        tl["bytes"] = [len(x) for x in tiles]
        tl["state"] = L.TILE_VALID
        w = e.window(1, t, np.zeros(0, np.uint32), tl, np.arange(len(t), dtype=np.int32))
        try:
            st = w.run(); res = w.results()
            parts = (w.task_entries().view(np.uint32) >> np.uint32(27)).astype(np.int64) + 1
        finally:
            w.close()
    # each CHECK ran as the parts its slices were planted for (the unit retires only after its last part)
    assert parts[:len(sizes)].tolist() == [part_cut(nb, pb)[0] for nb in sizes]
    if part_bytes >= 0:
        assert parts[3] == 32 and parts[0] > 1
    for i in range(len(sizes)):
        want = (counts[i] << 32) | int(tiles[i].view(np.uint32)[0])
        assert int(res["result"][i]) == want, (i, hex(int(res["result"][i])), hex(want))
    assert st["body_errors"] == sum(counts) and st["tasks_retired"] == len(t)
