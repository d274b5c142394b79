"""The NumPy restatement of the element-wise bodies (body_ref.py) against the sequential oracle, on random DTD programs
over every body at ragged sizes, and on the edge values of the float bodies; and a restatement of how wide tasks are cut
into parts and tiles into stage-in slices, which checks that the parts claim every slice that holds bytes.  No GPU."""
import numpy as np
import pytest

import body_ref as R
from parsec_b200 import _lib as L
from window_harness import run_oracle

EDGE_SIZES = [0, 1, 3, 4, 15, 16, 17, 4096 + 13]


def test_numpy_float32_keeps_denormals():
    d = R.bits_f32(R.DENORM)
    assert d != 0 and np.float32(d) + np.float32(d) == R.bits_f32(2 * R.DENORM)
    assert np.float32(1e-38) * np.float32(1e-3) != 0


def same_as_oracle(prog, layout):
    dag = prog.dag()
    ref = R.run_program(prog, layout)
    orc = run_oracle(dag, layout)
    assert np.array_equal(ref["result"], orc.res["result"]), "results"
    assert np.array_equal(ref["seen_version"], orc.res["seen_version"]), "seen versions"
    assert np.array_equal(ref["state"], orc.res["tiles"]["state"]), "tile states"
    assert np.array_equal(ref["version"], orc.res["tiles"]["version"]), "tile versions"
    for k in ("bytes_h2d", "bytes_d2h", "stage_ins", "body_errors"):
        assert ref["stats"][k] == orc.stats[k], (k, ref["stats"][k], orc.stats[k])
    diff = np.flatnonzero(ref["dev"] != orc.dev)
    assert not len(diff), f"{len(diff)} slab bytes differ, first at {diff[0]}"
    diff = np.flatnonzero(ref["host"] != orc.host)
    assert not len(diff), f"{len(diff)} host bytes differ, first at {diff[0]}"
    return ref


def random_case(seed, ntiles=30, ntasks=400):
    rng = np.random.default_rng(seed)
    sizes = list(EDGE_SIZES) + [int(v) for v in rng.integers(0, 4096 + 14, ntiles - len(EDGE_SIZES))]
    rng.shuffle(sizes)
    kinds = ["int"] * ntiles
    big = [i for i in range(ntiles - 1) if sizes[i] >= 64 and sizes[i + 1] >= 64]
    for i in big[:6:3]:                          # two fma pairs (x, y of unequal sizes)
        kinds[i], kinds[i + 1] = "fx", "fy"
    rest = [i for i in range(ntiles) if kinds[i] == "int"]
    for i in rest[::3]:
        kinds[i] = "float"
    layout = R.scattered_layout(rng, sizes, rng.random(ntiles) < 0.5)
    R.fill_kinds(rng, layout, kinds)
    return R.random_program(rng, sizes, ntasks, kinds), layout


@pytest.mark.parametrize("seed", range(6))
def test_random_programs_match_the_oracle(seed):
    prog, layout = random_case(seed)
    ref = same_as_oracle(prog, layout)
    bodies = {b for b, *_ in prog.tasks}
    assert bodies == set(range(14)), sorted(set(range(14)) - bodies)
    assert ref["stats"]["stage_ins"] > 0 and ref["stats"]["bytes_d2h"] > 0 and ref["stats"]["body_errors"] > 0


def edge_layout(rng, sizes):
    return R.scattered_layout(rng, sizes, np.ones(len(sizes), bool))


def test_float_edge_values_match_the_oracle():
    rng = np.random.default_rng(7)
    edge = np.array([0.0, -0.0, R.bits_f32(1), -R.bits_f32(0x7FFFFF), R.bits_f32(0x00800000), np.inf, -np.inf,
                     1.0, -3.5], np.float32)
    n = 4 * len(edge) * len(edge)
    layout = edge_layout(rng, [n + 3, n + 1, n, 37, 37, 64])
    # INCR_F32: every edge value plus every edge step but an infinity (+inf + -inf would make a NaN)
    R.put_words(layout, 0, np.repeat(edge, len(edge)))
    # AXPY x * k + y over every (x, y) edge pair: denormal and zero products meet zero or denormal y only, so that the
    # float64 sum is exact; an infinite product never meets an infinite y
    x, y = np.meshgrid(edge, edge, indexing="ij")
    x, y = x.reshape(-1).copy(), y.reshape(-1).copy()
    tiny_x, tiny_y = np.abs(x) < 2 ** -100, np.abs(y) < 2 ** -100
    x[tiny_x & ~tiny_y] = 0.0
    y[~tiny_x & tiny_y & np.isfinite(x) & (x != 0)] = -0.0
    bad = np.isinf(x) & np.isinf(y)
    y[bad] = 2.0
    R.put_words(layout, 1, x)
    R.put_words(layout, 2, y)
    prog = R.Program(6)
    for k in (0.0, -0.0, R.bits_f32(1), 1.0, -0.0, R.bits_f32(0x80000005)):
        prog.task(L.BODY_INCR_F32, [(0, L.ACCESS_RW)], fparam=k)
    prog.task(L.BODY_AXPY_F32, [(1, L.ACCESS_READ), (2, L.ACCESS_RW)], fparam=-1.5)
    prog.task(L.BODY_AXPY_F32, [(1, L.ACCESS_READ), (2, L.ACCESS_RW)], fparam=-0.5)   # the sign of the first: an infinity stays one
    # FILL_F32 stores the bits of NaN payloads and -0.0; CHECK_F32 tells -0.0 from +0.0 and one NaN from another
    for t, (fill, check) in enumerate([(R.QNAN, R.QNAN), (R.QNAN, R.QNAN_NEG), (R.NEG_ZERO, 0), (R.NEG_ZERO, R.NEG_ZERO)]):
        prog.task(L.BODY_FILL_F32, [(3 + t % 2, L.ACCESS_WRITE)], fparam=R.bits_f32(fill))
        prog.task(L.BODY_CHECK_F32, [(3 + t % 2, L.ACCESS_READ)], fparam=R.bits_f32(check))
    ref = same_as_oracle(prog, layout)
    checks = ref["result"][-8:][1::2]
    assert [int(r) >> 32 for r in checks] == [0, 9, 9, 0]
    assert [int(r) & 0xFFFFFFFF for r in checks] == [R.QNAN, R.QNAN, R.NEG_ZERO, R.NEG_ZERO]


def test_axpy_data_needs_fma():
    """On the fma pairs of the random programs, fma(k, x, y) and round(round(k * x) + y) differ often enough that a body
    computing the latter fails."""
    rng = np.random.default_rng(3)
    x, y, k = R.fma_pair_values(rng, 4096)
    fused = R.fma_f32(k, x, y)
    twice = (np.float32(k) * x) + y
    assert np.mean(fused != twice) >= 0.05


# ----------------------------------------------------------------------------------------------------------------------
# parts and stage-in slices (pb2_window_layout.h task_parts / stage_slice, pb2_sched.cuh part_slice, slices_over,
# tile_slices_of, live_slices)
# ----------------------------------------------------------------------------------------------------------------------
MAX_PARTS = 512
DEFAULT_SLICE = 64 * 1024


def task_parts(widest, part_bytes):
    return max(1, min(-(-widest // part_bytes), MAX_PARTS))


def stage_slice(slice_bytes, part_bytes):
    return slice_bytes if slice_bytes > 0 and (part_bytes <= 0 or slice_bytes < part_bytes) else part_bytes


def part_slice(widest, nparts, part, nbytes):
    per = (widest // nparts + 15) & ~15
    off = min(per * part, nbytes)
    ln = nbytes - off if part == nparts - 1 else (per if off + per <= nbytes else nbytes - off)
    return off, ln


def tile_slices(slice_bytes, nbytes):
    return max(1, min(-(-nbytes // slice_bytes), MAX_PARTS))


def slice_size(nbytes, ns):
    return (nbytes // ns + 15) & ~15


def live_slices(nbytes, ns):
    sper = slice_size(nbytes, ns)
    return ns if sper == 0 else min(ns, -(-nbytes // sper))


def slices_over(nbytes, ns, off, ln):
    sper = slice_size(nbytes, ns)
    s0 = min(off // sper, ns - 1)
    s1 = min((off + ln + sper - 1) // sper, ns)
    return (s0, s0) if ln == 0 else (s0, s1)


def claimed(nbytes, widest, part_bytes, slice_bytes=DEFAULT_SLICE):
    """(slices the parts of a task claim, the slices stage_in_slices waits for) of a tile of nbytes read by a task whose
    widest tile has `widest` bytes."""
    ns = tile_slices(stage_slice(slice_bytes, part_bytes), nbytes)
    npt = task_parts(widest, part_bytes)
    got = set()
    for p in range(npt):
        off, ln = part_slice(widest, npt, p, nbytes)
        s0, s1 = slices_over(nbytes, ns, off, ln)
        got.update(range(s0, s1))
    return got, ns


def test_finding_sizes_have_empty_slices():
    """Two tiles whose trailing slices are empty: the tile is complete with the slices that hold bytes."""
    for nbytes, pb in ((512 * 4097, 4096), (171, 18)):
        ns = tile_slices(stage_slice(DEFAULT_SLICE, pb), nbytes)
        assert (ns - 1) * slice_size(nbytes, ns) >= nbytes
        got, _ = claimed(nbytes, nbytes, pb)
        assert got == set(range(live_slices(nbytes, ns))) and live_slices(nbytes, ns) < ns


@pytest.mark.parametrize("pb", [4096, 16384])
def test_parts_claim_every_slice_that_holds_bytes(pb):
    """The completion target of stage_in_slices (live_slices) is the number of slices that hold a byte of the tile: the
    parts claim exactly those (else the tile never turns VALID, or turns VALID before its last slice is in)."""
    n = np.arange(512 * pb, 512 * pb + (4 << 20), 4, dtype=np.int64)     # every size cut into 512 parts and slices
    ns = np.minimum(-(-n // stage_slice(DEFAULT_SLICE, pb)), MAX_PARTS)
    sper = (n // ns + 15) & ~15
    holding = np.minimum((n - 1) // sper + 1, ns)          # slices up to the one that holds the last byte
    empty = np.flatnonzero(holding < ns)                  # sizes whose trailing slices are empty
    assert len(empty) > 0 if pb == 4096 else len(empty) == 0
    rng = np.random.default_rng(pb)
    sample = np.concatenate([n[rng.choice(empty, 40)] if len(empty) else n[:0], n[rng.choice(len(n), 40)]])
    for nbytes in sample.tolist():
        target = live_slices(nbytes, tile_slices(pb, nbytes))
        assert target == holding[(nbytes - n[0]) // 4]
        got, _ = claimed(nbytes, nbytes, pb)
        assert got == set(range(target)), nbytes


@pytest.mark.parametrize("part_bytes", [18, 100, 4096, 256 * 1024])
def test_parts_of_a_wider_task_claim_every_slice(part_bytes):
    """A tile read by a task whose widest flow is another tile is cut at that tile's offsets."""
    rng = np.random.default_rng(part_bytes)
    for _ in range(300):
        nbytes = int(rng.integers(1, 3 << 20))
        widest = nbytes + int(rng.integers(0, 1 << 20))
        got, ns = claimed(nbytes, widest, part_bytes)
        assert got == set(range(live_slices(nbytes, ns))), (nbytes, widest)
