"""GEMM windows checked bit for bit against a float64 evaluation and the sequential oracle.

Exact regime: operands in {-1, 0, +1} and C in small integers, sparse enough that every value a GEMM task reads or
writes is an integer of magnitude <= 256 and every partial sum of a task is bounded by 256 as well.  fp32 sums of such
values are exact in any order and every bf16 rounding is exact, so the fused chains (mode 0), the per-task units (modes
2 and 1) and the oracle must all produce the float64 result exactly.  Each case first checks that property on its own
data (oracle == float64, and a stated share of the GEMM contributions is nonzero), so a bad seed fails loudly instead
of loosening the comparison.

Tiles live in slots larger than their operand, at 16-byte but not 128-byte aligned addresses.  Operand padding and the
gaps between slots hold bf16 NaN, so a read past an operand shows up in C; C padding and the bytes after it hold a NaN
of another payload that must come back unchanged.  Besides the values, every run must match the oracle's bookkeeping:
dependency order, seen versions, tile versions, retired tasks, bytes moved, and the host image after pushout byte for
byte, padding included."""
import dataclasses
import functools

import numpy as np
import pytest

from oracle import orc
from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200.bf16 import bf16_bits_to_f32, f32_to_bf16_bits, round_to_bf16
from parsec_b200.engine import Engine
from parsec_b200.multigpu import cholesky_global
from window_harness import Layout, assert_like_oracle, placed, run_engine, run_oracle

pytestmark = pytest.mark.gpu

NAN = 0x7FC0            # operand padding and the gaps after operand slots
SENT = 0x7FA5           # C padding and the gap after a C slot (a NaN with another payload)
HOSTPAD = 0x1234        # host copy of a resident C tile's padding, different from its device padding
ONES = 0x3F803F80       # FILL_I32 pattern: two bf16 1.0
EXACT_MAX = 256         # every integer of magnitude <= 256 is a bf16 value


@pytest.fixture(scope="module")
def engines():
    made = {}

    def get(mode):
        if mode not in made:
            made[mode] = Engine(0, gemm_mode=mode, timeout_ms=4000)
        return made[mode]

    yield get
    for e in made.values():
        e.close()


def bits(x):
    return f32_to_bf16_bits(np.asarray(x, np.float32))


def ternary(rng, shape, p):
    """Entries in {-1, 0, +1}, nonzero with probability p."""
    sign = np.where(rng.random(shape) < 0.5, -1.0, 1.0)
    return np.where(rng.random(shape) < p, sign, 0.0)


def density(K):
    """About six nonzero products per dot product (two for the shortest K)."""
    return min(0.5, float(np.sqrt(6.0 / K)))


# ----------------------------------------------------------------------------------------------------------------------
# a window under construction: tiles with their contents and padding, tasks in insertion order, DTD dependencies
# ----------------------------------------------------------------------------------------------------------------------
class Win:
    def __init__(self):
        self.tiles = []                  # dict(data=u8 contents, pad, fill, valid, host_fill)
        self.flows = []                  # per task: [(tile, op)]
        self.rows = []                   # per task: (body, access list, iparam, fparam)

    def tile(self, values, pad=34, valid=False, c=False, host_pad=None):
        """values: 2-D float array (bf16-exact) or raw uint8 bytes, followed by `pad` bytes of padding in the tile: NaN
        for operands, SENT for C tiles (c=True), on the device and in the host copy unless host_pad says otherwise."""
        data = values if values.dtype == np.uint8 else bits(values).reshape(-1).view(np.uint8)
        fill = SENT if c else NAN
        self.tiles.append(dict(data=data.copy(), pad=pad, fill=fill, valid=valid,
                               host_fill=fill if host_pad is None else host_pad))
        return len(self.tiles) - 1

    def task(self, body, flows, iparam=(0, 0, 0), fparam=0.0):
        """flows: [(tile, access)] with access an engine access word (READ, RW, WRITE, | PUSHOUT)."""
        op = {L.ACCESS_READ: orc.DTD_INPUT, L.ACCESS_WRITE: orc.DTD_OUTPUT, L.ACCESS_RW: orc.DTD_INOUT}
        self.flows.append([(t, op[a & L.ACCESS_RW]) for t, a in flows])
        self.rows.append((body, [(t, a) for t, a in flows], iparam, fparam))
        return len(self.rows) - 1

    def gemm(self, a, b, c, M, N, K, pushout=False):
        return self.task(L.BODY_GEMM_BF16, [(a, L.ACCESS_READ), (b, L.ACCESS_READ),
                                            (c, L.ACCESS_RW | (L.FLOW_PUSHOUT if pushout else 0))], (M, N, K))

    def finish(self):
        """DTD dependencies (counter mode, orc_dtd.c), slab and host images."""
        n = len(self.rows)
        t = np.zeros(n, L.TASK_DTYPE)
        t["tile"][:] = -1
        ft = np.full((n, 4), -1, np.int32)
        fo = np.zeros((n, 4), np.int32)
        for i, (body, fl, ip, fp) in enumerate(self.rows):
            t["body"][i], t["nb_flows"][i], t["iparam"][i], t["fparam"][i] = body, len(fl), ip, fp
            for f, (tile, acc) in enumerate(fl):
                t["tile"][i, f], t["access"][i, f] = tile, acc
                ft[i, f], fo[i, f] = self.flows[i][f]
        src, dst, flow, dep = orc.dtd_build(t["nb_flows"].astype(np.int32), ft, fo, len(self.tiles))
        begin, count, succ = dags._csr_from_edges(n, src, dst, flow)
        t["succ_begin"], t["succ_count"], t["dep_goal"] = begin, count, dep
        return Case(t, succ, np.nonzero(dep == 0)[0].astype(np.int32), self.tiles)


def fill_u8(pattern, nbytes):
    return np.resize(np.array([pattern], np.uint16).view(np.uint8), nbytes)


class Case:
    """A window's arrays and its initial slab and host images.  Slot i of the slab starts at 16 mod 128 and holds tile i
    (values, then padding) followed by a gap of at least 48 bytes."""

    def __init__(self, tasks, succ, ready, tiles):
        self.tasks, self.succ, self.ready = tasks, np.asarray(succ, np.uint32), np.asarray(ready, np.int32)
        nt = len(tiles)
        self.bytes = np.array([len(x["data"]) + x["pad"] for x in tiles], np.int64)
        self.valid = np.array([x["valid"] for x in tiles], bool)
        self.doff, self.hoff = np.zeros(nt, np.int64), np.zeros(nt, np.int64)
        d, h = 16, 0
        for i in range(nt):
            self.doff[i], self.hoff[i] = d, h
            d = (d + int(self.bytes[i]) + 48 + 127) // 128 * 128 + 16
            h = (h + int(self.bytes[i]) + 15) // 16 * 16
        self.dev = fill_u8(NAN, d)
        self.host = np.zeros(max(h, 16), np.uint8)
        self.gap = np.ones(d, bool)             # bytes of the slab that belong to no tile
        for i, x in enumerate(tiles):
            n, o, ho = len(x["data"]), int(self.doff[i]), int(self.hoff[i])
            end = int(self.doff[i + 1]) if i + 1 < nt else d
            self.dev[o:end] = fill_u8(x["fill"], end - o)
            self.dev[o:o + n] = x["data"]
            self.host[ho:ho + n] = x["data"]
            self.host[ho + n:ho + int(self.bytes[i])] = fill_u8(x["host_fill"], x["pad"])
            self.gap[o:o + int(self.bytes[i])] = False
        self.dag = dags.Dag(self.tasks, self.succ, self.ready, ntiles=nt, tile_bytes=0, kind=1)
        self.layout = Layout(self.doff, self.hoff, self.bytes, self.valid, self.dev, self.host)

    def c_values(self, image, tile, M, N, host=False):
        o = int((self.hoff if host else self.doff)[tile])
        return bf16_bits_to_f32(image[o:o + M * N * 2].view(np.uint16)).reshape(M, N).astype(np.float64)


def topo_order(case):
    n = len(case.tasks)
    src, dst, _ = case.dag.edges()
    indeg = np.bincount(dst, minlength=n)
    adj = [[] for _ in range(n)]
    for s, d in zip(src, dst):
        adj[s].append(d)
    order, q = [], [i for i in range(n) if indeg[i] == 0]
    while q:
        i = q.pop(0)
        order.append(i)
        for d in adj[i]:
            indeg[d] -= 1
            if indeg[d] == 0:
                q.append(d)
    assert len(order) == n
    return order


def evaluate(case, launches=1, limit=EXACT_MAX):
    """Float64 evaluation of the window in a topological order, with the oracle's staging and pushout rules.  Asserts
    that every GEMM task only sees integers whose partial sums are bounded by `limit` in magnitude, in any order: with
    limit <= 256 every value is a bf16 value and the roundings are exact; with limit < 2^24 the fp32 sums are still
    exact, and the one rounding per task is round-to-nearest-even of an exact value.  Returns (slab image, host image,
    CHECK results) after the last launch, and the share of GEMM output elements whose product sum is nonzero."""
    dev, host = case.dev.copy(), case.host.copy()
    order = topo_order(case)
    result = np.zeros(len(case.tasks), np.uint64)
    nonzero, total = 0, 0
    for _ in range(launches):
        valid = case.valid.copy()
        for i in order:
            t = case.tasks[i]
            for f in range(t["nb_flows"]):
                k = int(t["tile"][f])
                if k >= 0 and t["access"][f] & L.ACCESS_READ and not valid[k]:
                    o, h, b = int(case.doff[k]), int(case.hoff[k]), int(case.bytes[k])
                    dev[o:o + b] = host[h:h + b]
                    valid[k] = True
            view = lambda f: dev[int(case.doff[t["tile"][f]]):][:int(case.bytes[t["tile"][f]])]
            if t["body"] == L.BODY_GEMM_BF16:
                M, N, K = (int(v) for v in t["iparam"])
                a = bf16_bits_to_f32(view(0)[:M * K * 2].view(np.uint16)).reshape(M, K).astype(np.float64)
                b = bf16_bits_to_f32(view(1)[:N * K * 2].view(np.uint16)).reshape(N, K).astype(np.float64)
                c = view(2)[:M * N * 2].view(np.uint16)
                c0 = bf16_bits_to_f32(c).reshape(M, N).astype(np.float64)
                p = a @ b.T
                out = c0 + p
                bound = np.abs(c0) + np.abs(a) @ np.abs(b).T
                assert bound.max() <= limit and np.array_equal(out, np.round(out)), "data outside the exact regime"
                nonzero += int(np.count_nonzero(p))
                total += p.size
                c[:] = bits(out).reshape(-1)
            elif t["body"] == L.BODY_COPY:
                n = min(len(view(0)), len(view(1)))
                view(1)[:n] = view(0)[:n]
            elif t["body"] == L.BODY_FILL_I32:
                v = view(0)
                v[:len(v) // 4 * 4].view(np.int32)[:] = t["iparam"][0]
            elif t["body"] == L.BODY_CHECK_I32:
                v = view(0)[:len(view(0)) // 4 * 4].view(np.int32)
                bad = int(np.count_nonzero(v != t["iparam"][0]))
                result[i] = np.uint64((bad << 32) | (int(v[0]) & 0xFFFFFFFF if len(v) else 0))
            else:
                assert t["body"] == L.BODY_NOP
            for f in range(t["nb_flows"]):
                k = int(t["tile"][f])
                if k >= 0 and t["access"][f] & L.ACCESS_WRITE:
                    valid[k] = True
                    if t["access"][f] & L.FLOW_PUSHOUT:
                        o, h, b = int(case.doff[k]), int(case.hoff[k]), int(case.bytes[k])
                        host[h:h + b] = dev[o:o + b]
    return dev, host, result, nonzero / max(total, 1)


def check_exact(case, ref, ref_f64, min_nonzero):
    """The data really is in the exact regime: the oracle's run `ref` equals the float64 evaluation, and enough GEMM
    products are nonzero for the comparison to mean something."""
    fdev, fhost, fres, share = ref_f64
    assert share >= min_nonzero, f"only {share:.2f} of the GEMM products are nonzero"
    assert np.array_equal(ref.dev, fdev), "oracle differs from the float64 evaluation on the device image"
    assert np.array_equal(ref.host, fhost), "oracle differs from the float64 evaluation on the host image"
    assert np.array_equal(ref.res["result"], fres)


def assert_matches(case, got, want):
    """One GPU run against the oracle's, and no byte between slots touched on the device."""
    assert np.array_equal(got.dev[case.gap], case.dev[case.gap]), "a byte between slots changed on the device"
    assert_like_oracle(got, want, case.dag)


# ----------------------------------------------------------------------------------------------------------------------
# 2, 3: shape sweep on padded tiles
# ----------------------------------------------------------------------------------------------------------------------
SHAPES = [
    (1, 8, 8),            # minimum shape; the second B box is wholly out of bounds
    (7, 264, 72),         # ragged rows; N % 16 == 8
    (129, 24, 1032),      # second row block; K tail
    (200, 520, 56),       # K < one k-block
    (1000, 1032, 136),    # 8 x 5 = 40 sub-tiles over 32 parts, non-square
    (64, 776, 8),         # N > 256 with M < 128
]


def sweep_case(M, N, K, seed, data):
    """One single task (resident C with pushout), a chain of 3 with pushout on the last member, and a chain of 3
    without pushout.  Pads vary and are not multiples of 16; some operands are resident, the others staged in."""
    rng = np.random.default_rng(seed)
    w = Win()
    pads = [34, 130, 6, 18 + 2 * N * 2, 258]
    pad = lambda: pads[len(w.tiles) % len(pads)]
    a = lambda: w.tile(data(rng, (M, K), "ab"), pad(), valid=len(w.tiles) % 3 == 1)
    b = lambda: w.tile(data(rng, (N, K), "ab"), pad(), valid=len(w.tiles) % 3 == 1)
    A, B = a(), b()
    C = w.tile(data(rng, (M, N), "c"), pad(), valid=True, c=True, host_pad=HOSTPAD)
    w.gemm(A, B, C, M, N, K, pushout=True)
    for pushout in (True, False):
        ops = [(a(), b()) for _ in range(3)]
        C = w.tile(data(rng, (M, N), "c"), pad(), c=True)
        for i, (A, B) in enumerate(ops):
            w.gemm(A, B, C, M, N, K, pushout=pushout and i == 2)
    return w.finish()


def exact_data(K):
    p = density(K)
    return lambda rng, shape, what: ternary(rng, shape, p) if what == "ab" else rng.integers(-3, 4, shape).astype(np.float64)


def realistic_data(rng, shape, what):
    return round_to_bf16((rng.uniform(-1, 1, shape) * 2.0 ** -6).astype(np.float32)).astype(np.float64)


@functools.lru_cache(maxsize=None)
def sweep_exact(M, N, K):
    return sweep_case(M, N, K, 7 * M + 11 * N + 13 * K, exact_data(K))


@functools.lru_cache(maxsize=None)
def sweep_refs(M, N, K):
    case = sweep_exact(M, N, K)
    return case, run_oracle(case.dag, case.layout), evaluate(case)


@pytest.mark.parametrize("mode", [0, 2, 1])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_shape_sweep_exact(engines, M, N, K, mode):
    case, ref_orc, ref_f64 = sweep_refs(M, N, K)
    check_exact(case, ref_orc, ref_f64, 0.3)
    assert_matches(case, run_engine(engines(mode), case.dag, case.layout), ref_orc)


def bf16_ulp(x):
    e = np.floor(np.log2(np.maximum(np.abs(x), 2.0 ** -126)))
    return 2.0 ** (e - 7)


@pytest.mark.parametrize("mode", [0, 2])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_shape_sweep_realistic(engines, M, N, K, mode):
    """Uniform bf16 data of magnitude 2^-6 against float64, element by element: one bf16 ulp of the largest partial
    value per rounding (the chains round once in mode 0 and once per member in mode 2), plus L*K * 2^-22 * sum|a b| for
    the fp32 accumulation of the L*K products, in whatever order the tensor core adds them."""
    case = sweep_case(M, N, K, 3 * M + 5 * N + K, realistic_data)
    st, res, dev, host, _, _ = run_engine(engines(mode), case.dag, case.layout)
    assert all(v == 0 for v in dags.check_execution(case.dag, res).values())
    # the three C tiles: tasks 0, 1..3, 4..6
    for members, pushout in (([0], True), ([1, 2, 3], True), ([4, 5, 6], False)):
        c_tile = int(case.tasks["tile"][members[0], 2])
        c = case.c_values(case.dev, c_tile, M, N)
        part, peak, absum = c.copy(), np.abs(c), np.zeros_like(c)
        for t in members:
            a = case.c_values(case.dev, int(case.tasks["tile"][t, 0]), M, K)
            b = case.c_values(case.dev, int(case.tasks["tile"][t, 1]), N, K)
            part = part + a @ b.T
            absum += np.abs(a) @ np.abs(b).T
            peak = np.maximum(peak, np.abs(part))
        roundings = 1 if mode == 0 else len(members)
        tol = roundings * bf16_ulp(peak) + len(members) * K * 2.0 ** -22 * absum
        for image, is_host in ((dev, False),) + (((host, True),) if pushout else ()):
            out = case.c_values(image, c_tile, M, N, host=is_host)
            err = np.abs(out - part)
            assert (err <= tol).all(), f"tile {c_tile}: {(err > tol).sum()} elements out of tolerance, max err {err.max()}"


def rounding_case(M, N, K, seed):
    """Single tasks (resident C with pushout, staged C without) whose exact integer results reach past 256, where bf16
    has no room for every integer: C0 in bf16 integers up to 2^12, dense ternary operands."""
    rng = np.random.default_rng(seed)
    w = Win()
    for valid, pushout in ((True, True), (False, False)):
        A, B = w.tile(ternary(rng, (M, K), 0.9)), w.tile(ternary(rng, (N, K), 0.9), valid=True)
        c0 = round_to_bf16(rng.integers(-4096, 4097, (M, N)).astype(np.float32)).astype(np.float64)
        C = w.tile(c0, pad=66, valid=valid, c=True, host_pad=HOSTPAD if valid else None)
        w.gemm(A, B, C, M, N, K, pushout=pushout)
    return w.finish()


@functools.lru_cache(maxsize=None)
def rounding_refs(M, N, K):
    case = rounding_case(M, N, K, M + N + K)
    return case, run_oracle(case.dag, case.layout), evaluate(case, limit=2 ** 24 - 1)


@pytest.mark.parametrize("mode", [0, 2])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_rounding_of_exact_sums(engines, M, N, K, mode):
    """The fp32 sums are exact and most results are not bf16 values: the kernel's one rounding per task must be the
    oracle's round-to-nearest-even, bit for bit."""
    case, ref_orc, ref_f64 = rounding_refs(M, N, K)
    check_exact(case, ref_orc, ref_f64, 0.5)
    c = [case.c_values(ref_f64[0], int(case.tasks["tile"][t, 2]), M, N) for t in range(2)]
    assert np.mean(np.abs(np.concatenate([x.ravel() for x in c])) > 256) > 0.5
    assert_matches(case, run_engine(engines(mode), case.dag, case.layout), ref_orc)


# ----------------------------------------------------------------------------------------------------------------------
# 5: DAGs that read GEMM outputs back as operands
# ----------------------------------------------------------------------------------------------------------------------
def readback_case(copies=256, seed=5):
    """Per copy: X (16 x 24) = C0 + A1 B1^T + A2 B2^T (a fusable chain); P += X Q^T (X as A); R += S X^T (X as B:
    N2 = 16, K2 = 24); Y = COPY(X), U += Y V^T; F = FILL(two bf16 1.0 per word), W += F Z^T; CHECK on P."""
    rng = np.random.default_rng(seed)
    w = Win()
    M, N, K = 16, 24, 40
    t = lambda shape, p=0.3, **kw: w.tile(ternary(rng, shape, p), pad=[6, 34, 130][len(w.tiles) % 3], **kw)
    c = lambda shape, **kw: w.tile(rng.integers(-2, 3, shape).astype(np.float64), pad=[18, 50][len(w.tiles) % 2], c=True, **kw)
    for i in range(copies):
        A1, B1, A2, B2 = t((M, K)), t((N, K), valid=True), t((M, K)), t((N, K))
        X = c((M, N))
        w.gemm(A1, B1, X, M, N, K)
        w.gemm(A2, B2, X, M, N, K)
        Q, P = t((32, N), 0.2), c((M, 32))
        w.gemm(X, Q, P, M, 32, N)
        S, R = t((40, N), 0.2, valid=True), c((40, M))
        w.gemm(S, X, R, 40, M, N, pushout=True)
        Y = c((M, N))
        w.task(L.BODY_COPY, [(X, L.ACCESS_READ), (Y, L.ACCESS_WRITE)])
        V, U = t((8, N), 0.2), c((M, 8))
        w.gemm(Y, V, U, M, 8, N, pushout=i % 2 == 0)
        F = w.tile(np.zeros(M * N * 2 + 2, np.uint8), pad=0)
        w.task(L.BODY_FILL_I32, [(F, L.ACCESS_WRITE)], (ONES, 0, 0))
        Z, Wt = t((8, N), 0.2), c((M, 8))
        w.gemm(F, Z, Wt, M, 8, N, pushout=True)
        w.task(L.BODY_CHECK_I32, [(P, L.ACCESS_READ)], (int(rng.integers(-2, 3)), 0, 0))
    return w.finish()


@functools.lru_cache(maxsize=None)
def readback_refs():
    case = readback_case()
    return case, run_oracle(case.dag, case.layout), evaluate(case)


@pytest.mark.parametrize("mode", [0, 2])
def test_readback_mixed_window(engines, mode):
    case, ref_orc, ref_f64 = readback_refs()
    check_exact(case, ref_orc, ref_f64, 0.3)
    got = run_engine(engines(mode), case.dag, case.layout)
    assert_matches(case, got, ref_orc)
    res = got.res
    # a GEMM output or a COPY / FILL result read back as an operand by a task on another worker (another SM)
    # (the operand flows of a GEMM only read, so every edge into them comes from the tile's last writer)
    src, dst, flow = case.dag.edges()
    readback = (case.tasks["body"][dst] == L.BODY_GEMM_BF16) & (flow < 2)
    assert readback.sum() == 4 * 256
    assert (res["worker"][src[readback]] != res["worker"][dst[readback]]).any(), "no read-back edge crossed workers"


def cholesky_case(NT, nb, seed):
    """cholesky_global on one GPU (POTRF a NOP), half of the tiles resident.  Without the panel solve the update DAG
    squares its values at every level, so only the last block row and the last two diagonal tiles start nonzero (about
    four nonzeros per row): TRSM(NT-1, NT-2) and the SYRK chain of T(NT-1, NT-1) then do nonzero work within the exact
    regime.  Every other task still adds its (zero) product into a C that later tasks read back as an operand."""
    tasks, succ, tiles, ready, _, _ = cholesky_global(NT, nb, 1, 1)
    rng = np.random.default_rng(seed)
    w = Win()
    for m in range(NT):
        for n in range(m + 1):
            live = m == NT - 1 or m == n == NT - 2
            i = len(w.tiles)
            w.tile(ternary(rng, (nb, nb), 4.0 / nb) if live else np.zeros((nb, nb)),
                   pad=[34, 130, 2 * nb * 2 + 6][i % 3], valid=i % 2 == 0, c=True)
    return Case(tasks, succ, ready, w.tiles)


@functools.lru_cache(maxsize=None)
def cholesky_refs(NT, nb):
    case = cholesky_case(NT, nb, 100 * NT + nb)
    return case, run_oracle(case.dag, case.layout), evaluate(case)


@pytest.mark.parametrize("mode", [0, 2])
@pytest.mark.parametrize("NT,nb", [(6, 128), (4, 264)])
def test_cholesky_exact(engines, NT, nb, mode):
    case, ref_orc, ref_f64 = cholesky_refs(NT, nb)
    check_exact(case, ref_orc, ref_f64, 0.02)
    assert_matches(case, run_engine(engines(mode), case.dag, case.layout), ref_orc)


# ----------------------------------------------------------------------------------------------------------------------
# 6: relaunch and a second window on the same engine and slab
# ----------------------------------------------------------------------------------------------------------------------
def test_relaunch_then_second_window(engines):
    engine = engines(0)
    first = sweep_exact(200, 520, 56)
    second = sweep_exact(7, 264, 72)
    ref1 = [run_oracle(first.dag, first.layout)]
    ref1.append(run_oracle(first.dag, dataclasses.replace(first.layout, dev=ref1[0].dev, host=ref1[0].host)))
    ref2 = run_oracle(second.dag, second.layout)
    check_exact(first, ref1[-1], evaluate(first, 2), 0.3)
    check_exact(second, ref2, evaluate(second, 1), 0.3)
    slab = engine.malloc(max(len(first.dev), len(second.dev)))
    try:
        with placed(engine, first.layout, slab=slab) as p:
            w = engine.window(1, first.tasks, first.succ, p.tiles, first.ready)
            try:
                runs = [p.run(w.run(), w.results()) for _ in range(2)]
            finally:
                w.close()
        # the second launch stages C in again from the pushed-out host copy: the oracle run twice
        assert not np.array_equal(runs[0].host, runs[1].host)
        for got, want in zip(runs, ref1):
            assert_matches(first, got, want)
        with placed(engine, second.layout, slab=slab) as p:
            w = engine.window(1, second.tasks, second.succ, p.tiles, second.ready)
            try:
                got = p.run(w.run(), w.results())
            finally:
                w.close()
        assert_matches(second, got, ref2)
    finally:
        engine.free(slab)


# ----------------------------------------------------------------------------------------------------------------------
# 7: window-creation refusals
# ----------------------------------------------------------------------------------------------------------------------
def refusal_base():
    w = Win()
    rng = np.random.default_rng(1)
    A, B = w.tile(ternary(rng, (16, 32), 0.3)), w.tile(ternary(rng, (24, 32), 0.3))
    C = w.tile(np.zeros((16, 24)), c=True)
    w.gemm(A, B, C, 16, 24, 32, pushout=True)
    return w


def refuse(kind):
    """The base window with one defect; returns (case, tiles hook, expected code, words of the message)."""
    w = refusal_base()
    hook = None
    if kind == "K%8":
        w.rows[0] = (w.rows[0][0], w.rows[0][1], (16, 24, 28), 0.0)
        code, msg = L.PB2_ERR_NOT_SUPPORTED, "K % 8"
    elif kind == "N%8":
        w.rows[0] = (w.rows[0][0], w.rows[0][1], (16, 20, 32), 0.0)
        code, msg = L.PB2_ERR_NOT_SUPPORTED, "N % 8"
    elif kind in ("M=0", "M<0"):
        w.rows[0] = (w.rows[0][0], w.rows[0][1], (0 if kind == "M=0" else -16, 24, 32), 0.0)
        code, msg = L.PB2_ERR_NOT_SUPPORTED, "M,N,K > 0"
    elif kind == "operand>tile":
        w.tiles[1]["data"], w.tiles[1]["pad"] = w.tiles[1]["data"][:-16], 14
        code, msg = L.PB2_ERR_VALUE_OUT_OF_BOUNDS, "operand larger"
    elif kind == "C>tile":
        w.tiles[2]["data"], w.tiles[2]["pad"] = w.tiles[2]["data"][:-2], 0
        code, msg = L.PB2_ERR_VALUE_OUT_OF_BOUNDS, "C larger"
    elif kind == "unaligned":
        hook = lambda t: t["dev_ptr"].__setitem__(0, t["dev_ptr"][0] + np.uint64(8))
        code, msg = L.PB2_ERR_BAD_PARAM, "16-byte aligned"
    elif kind == "two_shapes":
        C2 = w.tile(np.zeros((8, 24)), c=True)
        w.gemm(0, 1, C2, 8, 24, 32)
        code, msg = L.PB2_ERR_NOT_SUPPORTED, "two different operand shapes"
    elif kind == "2_flows":
        body, fl, ip, fp = w.rows[0]
        w.rows[0], w.flows[0] = (body, fl[:2], ip, fp), w.flows[0][:2]
        code, msg = L.PB2_ERR_BAD_PARAM, "3 data flows"
    else:
        assert kind == "no_C_tile"
        case = w.finish()
        case.tasks["tile"][0, 2] = -1
        return case, hook, L.PB2_ERR_BAD_PARAM, "3 data flows"
    return w.finish(), hook, code, msg


@pytest.mark.parametrize("kind", ["K%8", "N%8", "M=0", "M<0", "operand>tile", "C>tile", "unaligned", "two_shapes",
                                  "2_flows", "no_C_tile"])
def test_window_refusals(engines, kind):
    engine = engines(0)
    case, hook, code, msg = refuse(kind)
    slab = engine.malloc(len(case.dev) + 64)
    try:
        engine.h2d(slab, case.dev)
        host = case.host.copy()
        tiles = case.layout.table(slab, host.ctypes.data)
        if hook:
            hook(tiles)
        with pytest.raises(L.Pb2Error) as err:
            engine.window(1, case.tasks, case.succ, tiles, case.ready)
        assert err.value.rc == code and msg in str(err.value), str(err.value)
        # nothing ran: the slab and the host image are untouched, and the engine still runs a good window
        dev = np.empty_like(case.dev)
        engine.d2h(dev, slab)
        engine.synchronize()
        assert np.array_equal(dev, case.dev) and np.array_equal(host, case.host)
    finally:
        engine.free(slab)
    good = refusal_base().finish()
    assert_matches(good, run_engine(engine, good.dag, good.layout), run_oracle(good.dag, good.layout))
