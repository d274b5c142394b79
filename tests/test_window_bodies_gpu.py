"""Every element-wise body in HBM windows (pb2_hbm.cuh) and in the HBM-body units of GEMM windows (pb2_gemm.cuh)
against the NumPy reference (body_ref.py, window_ref.py): random DTD programs over ragged tiles whose slots sit at 16 mod 128 and whose
host homes are 16-, 4- and 1-byte aligned, with sentinel gaps between them; programs of producers followed by runs of
CHECK readers, which form read groups and fused producer units, and producers the planner must not fuse; both tile
movers, three part sizes (100 bytes leaves trailing parts and stage-in slices empty), groups fused, unfused or off, and
the engine's worker parameters; GEMM k-chains beside them in GEMM windows; and a window launched again over the
images its last run left.  Every run is compared with the reference on results, seen versions, final tile versions and
states, statistics, every byte of the slab and of the host image, and on an execution order that respects every edge."""
import dataclasses

import numpy as np
import pytest

import body_ref as B
import window_ref as R
from oracle import orc_dags as dags
from parsec_b200.engine import Engine
from window_harness import Run, fused, placed, run_engine, run_oracle

pytestmark = pytest.mark.gpu

SIZES = [0, 1, 3, 4, 15, 16, 17, 4096 + 12, 65536 + 4, (1 << 20) + 20]
GROUP_SIZES = [13, 4108, 40000, (1 << 20) + 20]
PART_BYTES = [0, 16384, 100]        # 0: the engine's default (256 KiB)
GROUPING = {"fused": {}, "unfused": dict(fuse_readers=-1), "nogroups": dict(read_groups=-1)}
REF_STATS = ("tasks_retired", "bytes_h2d", "bytes_d2h", "stage_ins", "body_errors")


@pytest.fixture(scope="module")
def engines():
    """engines(**params): one engine per parameter set for the module; set_part_bytes changes the part size per window."""
    made = {}

    def get(**kw):
        key = tuple(sorted(kw.items()))
        if key not in made:
            made[key] = Engine(0, **kw)
        return made[key]

    yield get
    for e in made.values():
        e.close()


# ----------------------------------------------------------------------------------------------------------------------
# programs and references, built once per module
# ----------------------------------------------------------------------------------------------------------------------
_CASES = {}


def cached(key, make):
    if key not in _CASES:
        _CASES[key] = make()
    return _CASES[key]


def every_body_case():
    """About 300 tasks over 40 tiles of SIZES and random sizes, every body, on a scattered layout."""
    def make():
        rng = np.random.default_rng(2024)
        nt = 40
        sizes = SIZES + [int(v) for v in rng.integers(0, 70000, nt - len(SIZES))]
        rng.shuffle(sizes)
        kinds = ["int"] * nt
        pairs = [i for i in range(nt - 1) if 64 <= sizes[i] and 64 <= sizes[i + 1]][:7:3]
        for i in pairs:
            kinds[i], kinds[i + 1] = "fx", "fy"
        for i in [i for i in range(nt) if kinds[i] == "int"][1::3]:
            kinds[i] = "float"
        layout = B.scattered_layout(rng, sizes, rng.random(nt) < 0.4)
        B.fill_kinds(rng, layout, kinds)
        prog = R.program(B.random_program(rng, sizes, 300, kinds))
        assert {b for b, *_ in prog.tasks} == set(range(14))
        copy_to = next(i for i in range(nt) if kinds[i] == "int" and sizes[i] > 4096)
        return dict(prog=prog, layout=layout, dag=prog.dag(), ref=R.run_program(prog, layout), copy_to=copy_to)
    return cached("every", make)


def grouped(size, staged):
    def make():
        prog, layout, episodes = R.grouped_case(size + int(staged), size, staged)
        return dict(prog=prog, layout=layout, episodes=episodes, dag=prog.dag(), ref=R.run_program(prog, layout))
    return cached(("grouped", size, staged), make)


def with_gemm(case, key):
    """The case's program with exact-regime GEMM k-chains appended, for GEMM windows."""
    def make():
        c = case()
        copy_to = c.get("copy_to", next(i for i, k in enumerate(c["layout"].nbytes) if k >= 4))
        prog, layout = R.with_gemm_chains(np.random.default_rng(7), c["prog"], c["layout"], copy_to)
        return dict(c, prog=prog, layout=layout, dag=prog.dag(kind=1), ref=R.run_program(prog, layout))
    return cached(("gemm",) + key, make)


# ----------------------------------------------------------------------------------------------------------------------
# running and comparing
# ----------------------------------------------------------------------------------------------------------------------
def run_window(eng, dag, layout, part_bytes):
    eng.set_part_bytes(part_bytes)
    return run_engine(eng, dag, layout)


def assert_like_ref(run, ref, dag):
    """One window run computes what the reference computes, in an order that respects every edge of dag; the first
    differing task or byte is reported."""
    bad = dags.check_execution(dag, run.res)
    assert all(v == 0 for v in bad.values()), bad
    diff = np.flatnonzero(run.res["result"] != ref["result"])
    assert not len(diff), (f"{len(diff)} results differ, first task {diff[0]} (body {dag.tasks['body'][diff[0]]}): "
                           f"{int(run.res['result'][diff[0]]):#x} != {int(ref['result'][diff[0]]):#x}")
    diff = np.flatnonzero(np.any(run.res["seen_version"] != ref["seen_version"], axis=1))
    assert not len(diff), f"{len(diff)} tasks saw other versions, first task {diff[0]}"
    for k in ("version", "state"):
        diff = np.flatnonzero(run.res["tiles"][k] != ref[k])
        assert not len(diff), f"tile {k} differs, first tile {diff[0]}"
    for k in REF_STATS:
        assert run.stats[k] == ref["stats"][k], (k, run.stats[k], ref["stats"][k])
    diff = np.flatnonzero(run.dev != ref["dev"])
    assert not len(diff), f"{len(diff)} slab bytes differ, first at {diff[0]}"
    diff = np.flatnonzero(run.host != ref["host"])
    assert not len(diff), f"{len(diff)} host bytes differ, first at {diff[0]}"


def gemm_unit(res, seq):
    """The tasks seq ran as one unit of a GEMM window: on one worker, each member's start and end consecutive events,
    the members one after the other (retire_unit_warp, pb2_gemm.cuh)."""
    ss, es = res["start_seq"].astype(np.int64), res["end_seq"].astype(np.int64)
    return (len(set(res["worker"][seq].tolist())) == 1 and np.array_equal(es[seq], ss[seq] + 1)
            and np.array_equal(ss[seq], ss[seq[0]] + 2 * np.arange(len(seq))))


def assert_fusion(res, episodes, kind=0):
    """Every episode the planner's rules fuse ran as one unit; every other one did not."""
    ran = (lambda p, m: fused(res, p, m)) if kind == 0 else (lambda p, m: gemm_unit(res, [p] + list(m)))
    for e in episodes:
        if e["fusable"]:
            assert ran(e["producer"], e["members"]), ("not fused", e)
        elif e["members"]:
            assert not ran(e["producer"], e["members"]), ("fused", e)
    assert sum(e["fusable"] for e in episodes) >= 8


# ----------------------------------------------------------------------------------------------------------------------
# 1. every body in an HBM window
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grouping", list(GROUPING))
@pytest.mark.parametrize("part_bytes", PART_BYTES)
@pytest.mark.parametrize("stage_mode", [0, 1])
def test_every_body_in_an_hbm_window(engines, stage_mode, part_bytes, grouping):
    c = every_body_case()
    run = run_window(engines(stage_mode=stage_mode, **GROUPING[grouping]), c["dag"], c["layout"], part_bytes)
    assert_like_ref(run, c["ref"], c["dag"])


@pytest.mark.parametrize("params", [dict(max_workers=1), dict(threads=32), dict(workers_per_sm=1),
                                    dict(queue_policy=1)], ids=lambda p: "%s=%d" % next(iter(p.items())))
def test_every_body_with_engine_parameters(engines, params):
    """One worker (fusion off: the FIFO order), 32-thread workers (the kernel is built for 64: every loop strides by
    blockDim.x), one worker per SM, and priority lanes with random priorities (the DTD edges make every order compute
    the same result)."""
    c = every_body_case()
    dag = c["dag"]
    if params.get("queue_policy"):
        dag = c["prog"].dag(priority=np.random.default_rng(1).integers(-5, 12, len(c["prog"].tasks)))
    run = run_window(engines(**params), dag, c["layout"], 16384)
    assert_like_ref(run, c["ref"], dag)


# ----------------------------------------------------------------------------------------------------------------------
# 2. read groups and fused producers in HBM windows
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grouping", list(GROUPING))
@pytest.mark.parametrize("part_bytes", PART_BYTES)
@pytest.mark.parametrize("stage_mode", [0, 1])
@pytest.mark.parametrize("staged", [False, True], ids=["resident", "staged"])
@pytest.mark.parametrize("size", GROUP_SIZES)
def test_grouped_program_in_an_hbm_window(engines, size, staged, stage_mode, part_bytes, grouping):
    c = grouped(size, staged)
    run = run_window(engines(stage_mode=stage_mode, **GROUPING[grouping]), c["dag"], c["layout"], part_bytes)
    assert_like_ref(run, c["ref"], c["dag"])
    if grouping == "fused":
        assert_fusion(run.res, c["episodes"])


# ----------------------------------------------------------------------------------------------------------------------
# 3. the same programs beside GEMM k-chains in GEMM windows
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grouping", ["fused", "unfused"])
@pytest.mark.parametrize("part_bytes", PART_BYTES)
@pytest.mark.parametrize("gemm_mode", [0, 2])
def test_every_body_in_a_gemm_window(engines, gemm_mode, part_bytes, grouping):
    """stage_mode 1 as well: the GEMM kernel moves tiles with its SIMT loops whatever the engine's mover."""
    c = with_gemm(every_body_case, ("every",))
    eng = engines(gemm_mode=gemm_mode, stage_mode=1, **GROUPING[grouping])
    run = run_window(eng, c["dag"], c["layout"], part_bytes)
    assert_like_ref(run, c["ref"], c["dag"])


@pytest.mark.parametrize("grouping", ["fused", "unfused"])
@pytest.mark.parametrize("part_bytes", PART_BYTES)
@pytest.mark.parametrize("gemm_mode", [0, 2])
@pytest.mark.parametrize("size", GROUP_SIZES)
def test_grouped_program_in_a_gemm_window(engines, size, gemm_mode, part_bytes, grouping):
    staged = GROUP_SIZES.index(size) % 2 == 1
    c = with_gemm(lambda: grouped(size, staged), ("grouped", size, staged))
    eng = engines(gemm_mode=gemm_mode, stage_mode=1, **GROUPING[grouping])
    run = run_window(eng, c["dag"], c["layout"], part_bytes)
    assert_like_ref(run, c["ref"], c["dag"])
    if grouping == "fused":
        assert_fusion(run.res, c["episodes"], kind=1)


# ----------------------------------------------------------------------------------------------------------------------
# 4. a window launched again over the images its last run left
# ----------------------------------------------------------------------------------------------------------------------
def relaunch(eng, dag, layout, launches):
    """`launches` runs of one window, waiting after each: [(stats, results, slab image, host image)] per run."""
    out = []
    with placed(eng, layout) as p:
        w = eng.window(dag.kind, dag.tasks, dag.succ, p.tiles, dag.ready)
        try:
            for _ in range(launches):
                st = w.run()
                res = w.results()
                dev, host = p.read()
                out.append((st, res, dev, host))
        finally:
            w.close()
    return out


def check_relaunch(eng, c, launches):
    """Run k computes what the program computes over the images run k - 1 left, from the tile table the window was
    created with (its states and versions).  The oracle confirms that expectation first, on the same images."""
    layout, dag = c["layout"], c["dag"]
    runs = relaunch(eng, dag, layout, launches)
    start = layout
    for k, (st, res, dev, host) in enumerate(runs):
        ref = R.run_program(c["prog"], start) if k else c["ref"]
        orc = run_oracle(dag, start)
        assert np.array_equal(orc.res["result"], ref["result"]) and np.array_equal(orc.dev, ref["dev"])
        assert np.array_equal(orc.host, ref["host"]) and np.array_equal(orc.res["tiles"]["version"], ref["version"])
        assert_like_ref(Run(st, res, dev, host, [], None), ref, dag)
        start = dataclasses.replace(layout, dev=dev, host=host)
    # the program is not idempotent: the runs computed different images
    assert not np.array_equal(runs[0][2], runs[1][2])


def test_relaunch_hbm_window(engines):
    """Three launches, so that both of the window's run-state copies are used."""
    eng = engines(stage_mode=0)
    eng.set_part_bytes(16384)
    check_relaunch(eng, every_body_case(), 3)


def test_relaunch_gemm_window(engines):
    """A GEMM window keeps one run-state copy."""
    eng = engines(gemm_mode=0, stage_mode=1)
    eng.set_part_bytes(0)
    check_relaunch(eng, with_gemm(every_body_case, ("every",)), 2)
