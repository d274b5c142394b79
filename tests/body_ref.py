"""A plain NumPy restatement of the element-wise task bodies 0-13 (the comments of enum pb2_body_e in
include/pb2_engine.h) and of a DTD program run over a slab and a host image, one task after the other.  The tests
compare the engine's kernels with it.

A flow is a uint8 view of its tile.  The 32-bit bodies see the whole 4-byte elements of a flow and leave its 1-3 tail
bytes alone; integers wrap modulo 2^32; INCR_F32 is a float32 add; AXPY is a fused multiply-add rounded once; CHECK
compares bits and returns mismatches << 32 | the flow's first element (0 when the flow has fewer than 4 bytes)."""
import dataclasses

import numpy as np

from oracle import orc
from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from window_harness import Layout

CHECKS = (L.BODY_CHECK_I32, L.BODY_CHECK_F32)


def f32_bits(x):
    return int(np.array([x], np.float32).view(np.uint32)[0])


def bits_f32(b):
    return np.array([b & 0xFFFFFFFF], np.uint32).view(np.float32)[0]


def words(flow):
    """The whole 4-byte elements of a uint8 flow, as a uint32 view that writes through."""
    return flow[:len(flow) // 4 * 4].view(np.uint32)


def fma_f32(k, x, y):
    """k * x + y for float32 arrays, rounded once to float32.  k * x is exact in float64, and the sum is asserted exact
    (TwoSum error 0) wherever it is finite, so the one rounding is the final float64 -> float32 conversion."""
    y64 = y.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        p = np.float64(np.float32(k)) * x.astype(np.float64)
        s = p + y64
        bb = s - p
        err = (p - (s - bb)) + (y64 - bb)
        fin = np.isfinite(s) & np.isfinite(p) & np.isfinite(y64)
        assert not np.any(err[fin]), "AXPY data whose float64 sum is not exact: the reference cannot round it once"
        return s.astype(np.float32)


def run_body(body, flows, iparam=(0, 0, 0), fparam=0.0):
    """Run one body in place on its flows (uint8 arrays); returns the task's result."""
    k = np.uint32(int(iparam[0]) & 0xFFFFFFFF)
    fk = np.float32(fparam)
    if body == L.BODY_NOP:
        return 0
    if body in CHECKS:
        e = words(flows[0])
        want = k if body == L.BODY_CHECK_I32 else fk.view(np.uint32)
        first = int(e[0]) if len(e) else 0
        return (int(np.count_nonzero(e != want)) << 32) | first
    if body == L.BODY_MEMSET_U8:
        flows[0][:] = int(iparam[0]) & 0xFF
        return 0
    if body == L.BODY_COPY:
        n = min(len(flows[0]), len(flows[1]))
        flows[1][:n] = flows[0][:n]
        return 0
    if body == L.BODY_AXPY_F32:
        n = min(len(flows[0]), len(flows[1])) // 4
        x = flows[0][:n * 4].view(np.float32)
        y = flows[1][:n * 4].view(np.float32)
        y[:] = fma_f32(fk, x, y)
        return 0
    e = words(flows[0])
    i = np.arange(len(e), dtype=np.uint32)
    with np.errstate(over="ignore"):
        if body == L.BODY_FILL_I32:
            e[:] = k
        elif body == L.BODY_FILL_F32:
            e[:] = fk.view(np.uint32)
        elif body == L.BODY_INCR_I32:
            e += k
        elif body == L.BODY_ADD_IOTA_I32:
            e += i
        elif body == L.BODY_SCALE_I32:
            e *= k
        elif body == L.BODY_IOTA_I32:
            e[:] = i
        elif body == L.BODY_INCR_F32:
            e.view(np.float32)[:] += fk
        elif body == L.BODY_ADD_AT_I32:
            at = int(iparam[0])
            if 0 <= at < len(e):
                e[at] += np.uint32(int(iparam[1]) & 0xFFFFFFFF)
        else:
            raise ValueError("not an element-wise body: %d" % body)
    return 0


# ----------------------------------------------------------------------------------------------------------------------
# DTD programs
# ----------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Program:
    """Tasks inserted in program order; each task is (body, [(tile, access word)], iparam, fparam).  Its DAG is what the
    DTD front end derives from the accesses (orc.dtd_build, counter mode)."""
    ntiles: int
    tasks: list = dataclasses.field(default_factory=list)

    def task(self, body, flows, iparam=(0, 0, 0), fparam=0.0):
        self.tasks.append((body, list(flows), tuple(int(v) for v in iparam), fparam))
        return len(self.tasks) - 1

    def dag(self):
        op = {L.ACCESS_READ: orc.DTD_INPUT, L.ACCESS_WRITE: orc.DTD_OUTPUT, L.ACCESS_RW: orc.DTD_INOUT}
        n = len(self.tasks)
        t = np.zeros(n, L.TASK_DTYPE)
        t["tile"][:] = -1
        ft = np.full((n, 4), -1, np.int32)
        fo = np.zeros((n, 4), np.int32)
        for i, (body, fl, ip, fp) in enumerate(self.tasks):
            t["body"][i], t["nb_flows"][i], t["iparam"][i] = body, len(fl), ip
            t["fparam"][i] = np.float32(fp)
            for f, (tile, acc) in enumerate(fl):
                t["tile"][i, f], t["access"][i, f] = tile, acc
                ft[i, f], fo[i, f] = tile, op[acc & L.ACCESS_RW]
        src, dst, flow, dep = orc.dtd_build(t["nb_flows"].astype(np.int32), ft, fo, self.ntiles)
        begin, count, succ = dags._csr_from_edges(n, src, dst, flow)
        t["succ_begin"], t["succ_count"], t["dep_goal"] = begin, count, dep
        return dags.Dag(t, succ, np.nonzero(dep == 0)[0].astype(np.int32), ntiles=self.ntiles, tile_bytes=0, name="dtd")


def run_program(prog, layout):
    """The program, task by task in program order, over copies of the layout's two images.  A READ of an INVALID tile
    stages it in from its home first; a WRITE-only flow does not stage, and leaves the tile VALID; a pushout flow copies
    the whole tile home after the body.  Returns dict(dev, host, result, seen_version, state, version, stats)."""
    dev, host = layout.dev.copy(), layout.host.copy()
    nt = len(layout.nbytes)
    valid = np.array(layout.valid, bool)
    version = np.zeros(nt, np.uint32)
    n = len(prog.tasks)
    result = np.zeros(n, np.uint64)
    seen = np.zeros((n, L.MAX_FLOWS), np.uint32)
    st = dict(bytes_h2d=0, bytes_d2h=0, stage_ins=0, body_errors=0, tasks_retired=n)

    def slot(i):
        return dev[int(layout.doff[i]):int(layout.doff[i]) + int(layout.nbytes[i])]

    def home(i):
        return host[int(layout.hoff[i]):int(layout.hoff[i]) + int(layout.nbytes[i])]

    for t, (body, fl, ip, fp) in enumerate(prog.tasks):
        for f, (i, acc) in enumerate(fl):
            seen[t, f] = version[i]
            if acc & L.ACCESS_READ and not valid[i]:
                slot(i)[:] = home(i)
                st["bytes_h2d"] += int(layout.nbytes[i])
                st["stage_ins"] += 1
                valid[i] = True
        r = run_body(body, [slot(i) for i, _ in fl], ip, fp)
        result[t] = r
        if body in CHECKS:
            st["body_errors"] += r >> 32
        for i, acc in fl:
            if acc & L.ACCESS_WRITE:
                version[i] += 1
                valid[i] = True
                if acc & L.FLOW_PUSHOUT:
                    home(i)[:] = slot(i)
                    st["bytes_d2h"] += int(layout.nbytes[i])
    state = np.where(valid, L.TILE_VALID, L.TILE_INVALID).astype(np.int32)
    return dict(dev=dev, host=host, result=result, seen_version=seen, state=state, version=version, stats=st)


def scattered_layout(rng, nbytes, valid, slab_fill=0xA5, host_fill=0x3C):
    """Tile i in a slab slot at 16 mod 128 followed by a gap of at least 48 sentinel bytes; its home in the host image at
    an offset that is 16-, 4- or 1-byte aligned (in turn), after a gap of at least 8 sentinel bytes.  Resident tiles
    hold random bytes in the slab and other random bytes at home; staged tiles hold random bytes at home and sentinels
    in the slab."""
    nbytes = np.asarray(nbytes, np.int64)
    nt = len(nbytes)
    doff, hoff = np.zeros(nt, np.int64), np.zeros(nt, np.int64)
    d, h = 16, 0
    for i in range(nt):
        doff[i] = d
        d = (d + int(nbytes[i]) + 48 + 127) // 128 * 128 + 16
        h = (h + 8 + 15) // 16 * 16 + (0, 4, 3)[i % 3]
        hoff[i] = h
        h += int(nbytes[i])
    dev = np.full(d, slab_fill, np.uint8)
    host = np.full(h + 16, host_fill, np.uint8)
    valid = np.asarray(valid, bool)
    for i in range(nt):
        n = int(nbytes[i])
        host[hoff[i]:hoff[i] + n] = rng.integers(0, 4, n, dtype=np.uint8)
        if valid[i]:
            dev[doff[i]:doff[i] + n] = rng.integers(0, 4, n, dtype=np.uint8)
    return Layout(doff, hoff, nbytes, valid, dev, host)


def put_words(layout, i, values, where="both"):
    """Store uint32/float32 values at the start of tile i, in the slab and/or at home."""
    b = np.ascontiguousarray(values).view(np.uint8)
    n = min(len(b), int(layout.nbytes[i]) // 4 * 4)
    if where in ("both", "dev"):
        layout.dev[int(layout.doff[i]):int(layout.doff[i]) + n] = b[:n]
    if where in ("both", "host"):
        layout.host[int(layout.hoff[i]):int(layout.hoff[i]) + n] = b[:n]


# ----------------------------------------------------------------------------------------------------------------------
# random programs over every body
# ----------------------------------------------------------------------------------------------------------------------
QNAN = 0x7FC01234         # quiet NaNs with payloads: FILL_F32 stores and CHECK_F32 compares their bits
QNAN_NEG = 0xFFC00042
NEG_ZERO = 0x80000000
DENORM = 0x00000003


def float_values(rng, n):
    """float32 values for the tiles float bodies add to: multiples of 1/16 in [-8, 8], with +-0, denormals and +-inf."""
    v = (rng.integers(-128, 129, n) / 16.0).astype(np.float32)
    edge = np.array([0.0, -0.0, bits_f32(DENORM), -bits_f32(0x000F0000), np.inf, -np.inf], np.float32)
    pick = rng.random(n) < 0.1
    v[pick] = edge[rng.integers(0, len(edge), int(pick.sum()))]
    return v


def fma_pair_values(rng, n):
    """(x, y, k): data where fma(k, x, y) and k * x + y rounded twice often differ, and the float64 sum is exact."""
    x = rng.uniform(1.0, 2.0, n).astype(np.float32)
    y = (-rng.uniform(1.0, 3.0, n)).astype(np.float32)
    return x, y, np.float32(rng.uniform(1.0, 2.0))


def random_program(rng, nbytes, ntasks, kinds, pushout=True):
    """A DTD program of ntasks tasks over the tiles, covering every body 0-13.  kinds[i] says what tile i holds: "int"
    (integer bodies, MEMSET, FILL_F32 / CHECK_F32 with NaN payloads and -0.0, COPY between int tiles), "float" (INCR_F32
    with finite steps, FILL_F32 and CHECK_F32, COPY between float tiles), or "fx" / "fy" (one fma pair: the x and the y
    tile of one AXPY, i and i + 1).  No float arithmetic ever meets a NaN, and no +inf meets a -inf."""
    nt = len(nbytes)
    ints = [i for i in range(nt) if kinds[i] == "int"]
    floats = [i for i in range(nt) if kinds[i] == "float"]
    pairs = [i for i in range(nt) if kinds[i] == "fx"]
    prog = Program(nt)

    def acc(base, i):
        return base | (L.FLOW_PUSHOUT if pushout and base & L.ACCESS_WRITE and rng.random() < 0.25 else 0)

    def filler():
        return L.ACCESS_WRITE if rng.random() < 0.5 else L.ACCESS_RW

    def two(pool):
        a, b = rng.choice(pool, 2, replace=False)
        return int(a), int(b)

    def f_const():
        return float(rng.choice([0.0, -0.0, float(bits_f32(DENORM)), 1.5, -2.25, 0.0625]))

    bodies = [L.BODY_NOP, L.BODY_FILL_I32, L.BODY_CHECK_I32, L.BODY_INCR_I32, L.BODY_ADD_IOTA_I32, L.BODY_SCALE_I32,
              L.BODY_IOTA_I32, L.BODY_COPY, L.BODY_FILL_F32, L.BODY_CHECK_F32, L.BODY_INCR_F32, L.BODY_MEMSET_U8,
              L.BODY_ADD_AT_I32]
    order = [bodies[j % len(bodies)] for j in range(ntasks)]
    rng.shuffle(order)
    axpy_at = {int(j): p for j, p in zip(rng.choice(ntasks, len(pairs), replace=False), pairs)}
    for j, body in enumerate(order):
        if j in axpy_at:
            x = axpy_at[j]
            _, _, k = fma_pair_values(rng, 1)
            prog.task(L.BODY_AXPY_F32, [(x, L.ACCESS_READ), (x + 1, acc(L.ACCESS_RW, x + 1))], fparam=k)
            continue
        i = int(rng.choice(ints))
        if body == L.BODY_NOP:
            prog.task(body, [(i, L.ACCESS_READ)])
        elif body in (L.BODY_FILL_I32, L.BODY_MEMSET_U8, L.BODY_IOTA_I32):
            prog.task(body, [(i, acc(filler(), i))], (int(rng.integers(0, 4)), 0, 0))
        elif body == L.BODY_CHECK_I32:
            prog.task(body, [(i, L.ACCESS_READ)], (int(rng.integers(0, 4)), 0, 0))
        elif body in (L.BODY_INCR_I32, L.BODY_ADD_IOTA_I32, L.BODY_SCALE_I32):
            prog.task(body, [(i, acc(L.ACCESS_RW, i))], (int(rng.integers(-3, 4)), 0, 0))
        elif body == L.BODY_ADD_AT_I32:
            n = int(nbytes[i]) // 4
            at = int(rng.choice([0, n - 1, n, n + 5, -1, int(rng.integers(0, max(n, 1)))]))
            prog.task(body, [(i, acc(L.ACCESS_RW, i))], (at, int(rng.integers(1, 1 << 30)), 0))
        elif body == L.BODY_COPY:
            a, b = two(floats if rng.random() < 0.4 else ints)
            prog.task(body, [(a, L.ACCESS_READ), (b, acc(filler(), b))])
        elif body == L.BODY_FILL_F32:
            if rng.random() < 0.5:
                prog.task(body, [(i, acc(filler(), i))], fparam=bits_f32(int(rng.choice([QNAN, QNAN_NEG, NEG_ZERO]))))
            else:
                x = int(rng.choice(floats))
                prog.task(body, [(x, acc(filler(), x))], fparam=f_const())
        elif body == L.BODY_CHECK_F32:
            pool = floats + pairs + [p + 1 for p in pairs] if rng.random() < 0.5 else ints
            x = int(rng.choice(pool))
            k = bits_f32(int(rng.choice([QNAN, QNAN_NEG, NEG_ZERO, 0, f32_bits(1.5)])))
            prog.task(body, [(x, L.ACCESS_READ)], fparam=k)
        elif body == L.BODY_INCR_F32:
            x = int(rng.choice(floats))
            prog.task(body, [(x, acc(L.ACCESS_RW, x))], fparam=f_const())
    return prog


def fill_kinds(rng, layout, kinds):
    """Give the float tiles and the fma pairs of a layout their values (slab and home)."""
    for i, kd in enumerate(kinds):
        n = int(layout.nbytes[i]) // 4
        if kd == "float":
            put_words(layout, i, float_values(rng, n))
        elif kd == "fx":
            x, y, _ = fma_pair_values(rng, n)
            put_words(layout, i, x)
            put_words(layout, i + 1, y)
