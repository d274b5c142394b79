"""Placing, running and checking engine windows, for the GPU tests.

A `Layout` says where a window's tiles live in a device slab and in their host home, and holds the images both start
from.  `placed` puts a layout on an engine for the duration of a `with` block, `run_engine` runs a DAG there once (or
several times), and `run_oracle` runs the sequential oracle (oracle/orc.py) on copies of the same two images.  Both
return a `Run`, and `assert_same_run` / `assert_like_oracle` compare two of them.

Where a tile sits selects device code paths (a host copy that is only 4- or 1-byte aligned takes the narrow copy loops,
DESIGN §5), so a test that moves a tile tests something else: the constructors below keep the layouts the tests have
always used."""
import contextlib
import dataclasses
from typing import NamedTuple

import numpy as np
import pytest

from oracle import orc
from oracle import orc_dags as dags
from parsec_b200 import _lib as L

STATS = ("tasks_retired", "bytes_h2d", "bytes_d2d", "bytes_d2h", "stage_ins", "body_errors")


def _starts(sizes):
    return np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)


@dataclasses.dataclass
class Layout:
    """Tile i has nbytes[i] bytes at byte doff[i] of the slab and at byte hoff[i] of the host image (hoff None: no tile
    has a host home, src_ptr 0), and starts VALID (resident in the slab) when valid[i], else INVALID (staged in from
    its home when first read).  dev and host are the images the window starts from."""
    doff: np.ndarray
    hoff: np.ndarray
    nbytes: np.ndarray
    valid: np.ndarray
    dev: np.ndarray
    host: np.ndarray

    @classmethod
    def packed(cls, dag, host=None, valid=False, sizes=None):
        """One slot per tile, rounded up to 512 bytes, in a slab of at least 16 bytes; the host copies back to back.
        sizes: bytes per tile (default dag.tile_bytes each); valid: every tile starts resident, holding its host bytes."""
        sz = np.full(dag.ntiles, dag.tile_bytes, np.int64) if sizes is None else np.asarray(sizes, np.int64)
        slots = (sz + 511) // 512 * 512
        return cls._fill(_starts(slots), max(int(slots.sum()), 16), sz, host, valid)

    @classmethod
    def contiguous(cls, dag, dev=None, host=None, valid=True):
        """Tile i at byte i * tile_bytes of the slab and of the host image.  dev: the slab's initial bytes (default
        zeros, or the host bytes of resident tiles)."""
        sz = np.full(dag.ntiles, dag.tile_bytes, np.int64)
        layout = cls._fill(_starts(sz), int(sz.sum()), sz, host, valid)
        if dev is not None:
            layout.dev[:] = np.asarray(dev).view(np.uint8).reshape(-1)
        return layout

    @classmethod
    def _fill(cls, doff, slab_bytes, sz, host, valid):
        nt = len(sz)
        hoff = None if host is None else _starts(sz)
        host = np.zeros(0, np.uint8) if host is None else np.asarray(host).view(np.uint8).reshape(-1).copy()
        dev = np.zeros(slab_bytes, np.uint8)
        valid = np.full(nt, bool(valid))
        for i in (np.flatnonzero(valid) if hoff is not None else ()):
            dev[doff[i]:doff[i] + sz[i]] = host[hoff[i]:hoff[i] + sz[i]]
        return cls(doff, hoff, sz, valid, dev, host)

    def table(self, dev_base, host_base):
        """The tile table of the window: the engine's for a slab and the device alias of the host image, the
        oracle's (orc.run_window_raw) for the addresses of its two images."""
        t = np.zeros(len(self.nbytes), L.TILE_DTYPE)
        t["dev_ptr"] = np.uint64(dev_base) + self.doff.astype(np.uint64)
        t["src_ptr"] = 0 if self.hoff is None else np.uint64(host_base) + self.hoff.astype(np.uint64)
        t["bytes"] = self.nbytes
        t["state"] = np.where(self.valid, L.TILE_VALID, L.TILE_INVALID)
        return t

    def offsets(self):
        """The table of orc.run_window and priority_order.replay: src_ptr is the byte offset of the home."""
        return self.table(0, 0)

    def tile_bytes(self, image, i):
        """Tile i's bytes in a slab image."""
        return image[int(self.doff[i]):int(self.doff[i]) + int(self.nbytes[i])]


class Run(NamedTuple):
    """One run of a window: stats, results (pb2_window_results, or the oracle's), the slab and host images after it,
    the trace of each launch (traced windows), and the final tile table with dev_ptr / src_ptr as offsets into the
    two images."""
    stats: dict
    res: dict
    dev: np.ndarray
    host: np.ndarray
    traces: list
    table: np.ndarray


def _rebased(tiles, dev_base, host_base):
    t = tiles.copy()
    t["dev_ptr"] -= np.uint64(dev_base)
    t["src_ptr"] = np.where(t["src_ptr"] != 0, t["src_ptr"] - np.uint64(host_base), 0)
    return t


@dataclasses.dataclass
class Placed:
    """A layout on an engine: the slab, the registered copy of the host image and its device alias, the tile table."""
    engine: object
    layout: Layout
    slab: int
    host: np.ndarray
    alias: int
    tiles: np.ndarray
    dev: np.ndarray = None

    def read(self):
        """(slab image, host image) now."""
        dev = self.engine.d2h(np.empty_like(self.layout.dev), self.slab)
        self.engine.synchronize()
        return dev, self.host.copy()

    def run(self, stats, res, traces=(), images=None):
        """The Run of a window over this placement with these stats and results, and the images now (or `images`)."""
        dev, host = self.read() if images is None else images
        return Run(stats, res, dev, host, list(traces), _rebased(res["tiles"], self.slab, self.alias))


@contextlib.contextmanager
def placed(engine, layout, slab=None):
    """Places `layout` on `engine` (in `slab` if given, else in a fresh one it frees): uploads the slab image and
    registers a copy of the host image.  After the block, .dev and .host hold the final images."""
    own = slab is None
    slab = engine.malloc(len(layout.dev)) if own else slab
    host = layout.host.copy()
    registered = False
    try:
        engine.h2d(slab, layout.dev)
        alias = 0
        if layout.hoff is not None:
            alias = engine.host_register(host)
            registered = True
        p = Placed(engine, layout, slab, host, alias, layout.table(slab, alias))
        yield p
        p.dev, p.host = p.read()
    finally:
        if registered:
            engine.host_unregister(host)
        if own:
            engine.free(slab)


def run_engine(engine, dag, layout, launches=1, trace=False):
    """`launches` runs of one window of dag over `layout` on engine; the Run of the last one (traces: every launch's)."""
    assert layout.hoff is not None or not np.any(dag.tasks["access"] & L.FLOW_PUSHOUT), "pushout without a host home"
    with placed(engine, layout) as p:
        if trace:
            engine.set_window_trace(True)
        try:
            w = engine.window(dag.kind, dag.tasks, dag.succ, p.tiles, dag.ready)
        finally:
            if trace:
                engine.set_window_trace(False)
        try:
            traces = []
            for _ in range(launches):
                st = w.run()
                if trace:
                    traces.append(w.trace())
            res = w.results()
        finally:
            w.close()
    return p.run(st, res, traces, (p.dev, p.host))


def run_oracle(dag, layout):
    """The sequential oracle (FIFO ready order) on copies of the layout's two images."""
    dev, host = layout.dev.copy(), layout.host.copy()
    r = orc.run_window_raw(dag.tasks, dag.succ, layout.table(dev.ctypes.data, host.ctypes.data), dag.ready)
    assert r["rc"] == 0
    return Run(r["stats"], r, dev, host, [], _rebased(r["tiles"], dev.ctypes.data, host.ctypes.data))


def assert_same_run(a, b, stats=STATS):
    """Two runs of one window compute the same thing: results, seen versions, tile table, both images, stats."""
    for k in ("result", "seen_version"):
        assert np.array_equal(a.res[k], b.res[k]), k
    assert a.table.tobytes() == b.table.tobytes(), "tile table"
    assert np.array_equal(a.dev, b.dev), "slab image"
    assert np.array_equal(a.host, b.host), "host image"
    for k in stats:
        assert a.stats[k] == b.stats[k], (k, a.stats[k], b.stats[k])


def assert_like_oracle(run, ref, dag, stats=STATS):
    """A run computes what the oracle's run `ref` computes, in an order that respects every edge of dag."""
    bad = dags.check_execution(dag, run.res)
    assert all(v == 0 for v in bad.values()), bad
    for k in ("result", "seen_version"):
        assert np.array_equal(run.res[k], ref.res[k]), k
    for k in ("version", "state"):
        assert np.array_equal(run.res["tiles"][k], ref.res["tiles"][k]), "tile " + k
    for k in stats:
        assert run.stats[k] == ref.stats[k], (k, run.stats[k], ref.stats[k])
    diff = np.flatnonzero(run.dev != ref.dev)
    assert not len(diff), f"{len(diff)} slab bytes differ from the oracle's, first at {diff[0]}"
    diff = np.flatnonzero(run.host != ref.host)
    assert not len(diff), f"{len(diff)} host bytes differ from the oracle's, first at {diff[0]}"


# ----------------------------------------------------------------------------------------------------------------------
# fused units: a producer and the readers of the tile it writes, run with fusion on and off
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def engines():
    from parsec_b200.engine import Engine
    with Engine(0) as on, Engine(0, fuse_readers=-1) as off:
        yield on, off


def check_pair(engines, dag, layout):
    """dag on both engines of a pair: the same run, and the oracle's.  Returns the two results."""
    a, b = (run_engine(e, dag, layout) for e in engines)
    assert_same_run(a, b)
    ref = run_oracle(dag, layout)
    assert_like_oracle(a, ref, dag)
    assert_like_oracle(b, ref, dag)
    return a.res, b.res


def readers_dag(producer_body, producer_k, reader_ks, tile_bytes, access=L.ACCESS_WRITE):
    """Task 0 writes tile 0 (FILL k / IOTA), tasks 1.. read it with CHECK constants reader_ks (ints: CHECK_I32, floats:
    CHECK_F32 with those bits)."""
    n = 1 + len(reader_ks)
    t = np.zeros(n, L.TASK_DTYPE)
    t["tile"][:] = -1
    t["nb_flows"] = 1
    t["tile"][:, 0] = 0
    t["body"][0], t["iparam"][0, 0], t["access"][0, 0] = producer_body, producer_k, access
    for i, k in enumerate(reader_ks, start=1):
        t["access"][i, 0] = L.ACCESS_READ
        t["dep_goal"][i] = 1
        if isinstance(k, float):
            t["body"][i], t["fparam"][i] = L.BODY_CHECK_F32, np.float32(k)
        else:
            t["body"][i], t["iparam"][i, 0] = L.BODY_CHECK_I32, k
    t["succ_begin"][0], t["succ_count"][0] = 0, n - 1
    t["succ_begin"][1:] = n - 1
    succ = np.arange(1, n, dtype=np.uint32)
    return dags.Dag(t, succ, np.array([0], np.int32), ntiles=1, tile_bytes=tile_bytes, name="readers")


f5 = float(np.array([5], np.int32).view(np.float32)[0])     # a CHECK_F32 constant whose bits are the integer 5
KS = [5, 5, 6, f5, 0, 7, 1, 5]


def fused(res, p, members):
    """The members ran in p's unit: on p's worker, started right after p ended, in member order."""
    ss, es = res["start_seq"].astype(np.int64), res["end_seq"].astype(np.int64)
    return all(res["worker"][m] == res["worker"][p] and ss[m] == es[p] + 1 + i for i, m in enumerate(members))


def not_fused(res, p, members):
    """The group ran as a task of its own.  (A group popped from the ring by p's own worker right after p, with no other
    event in between, would look fused; with every worker polling the ring that does not happen.)"""
    return not fused(res, p, members)
