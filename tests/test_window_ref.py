"""The window reference (window_ref.py) against the sequential oracle, with no GPU: programs whose producers and CHECK
readers form read groups and fused units, the restated read-group rules on a hand-made DAG, GEMM k-chains beside
every element-wise body, and the exactness assertion of the GEMM reference."""
import numpy as np
import pytest

import window_ref as R
from parsec_b200 import _lib as L
from parsec_b200.bf16 import bf16_bits_to_f32, f32_to_bf16_bits
from test_body_ref import random_case
from window_harness import run_oracle


def same_as_oracle(prog, layout):
    """The reference and the oracle agree on every result, version, state, statistic and byte (as test_body_ref)."""
    ref = R.run_program(prog, layout)
    orc = run_oracle(prog.dag(), layout)
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


# ----------------------------------------------------------------------------------------------------------------------
# programs that form read groups and fused units, and GEMM k-chains beside element-wise programs
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("staged", [False, True])
@pytest.mark.parametrize("size", [13, 4108])
def test_grouped_programs_match_the_oracle(size, staged):
    prog, layout, episodes = R.grouped_case(size, size, staged)
    ref = same_as_oracle(prog, layout)
    assert {e["kind"] for e in episodes} == set(R.EPISODES)
    fusable = [e for e in episodes if e["fusable"]]
    assert len(fusable) >= 16 and len(episodes) - len(fusable) >= 6
    assert all(len(e["members"]) >= 2 for e in episodes if e["fusable"])
    # passing and failing constants, a failing leader among the fused units
    res = ref["result"]
    assert any(res[e["members"][0]] >> 32 for e in fusable) and any(not res[e["members"][0]] >> 32 for e in fusable)


def test_read_groups_restate_the_planner_rules():
    """Hand-made cases of read_groups: a NOP splits a run, the first group of at least two fuses, a wider read tile, a
    COPY of unequal sizes and a pushout of X refuse fusion, a run longer than GROUP_MAX is cut."""
    nbytes = np.array([64, 64, 32, 128])
    prog = R.Program(4)
    prog.task(L.BODY_FILL_I32, [(0, L.ACCESS_WRITE), (2, L.ACCESS_READ)])             # 0: fuses with 3, 4
    prog.task(L.BODY_CHECK_I32, [(0, L.ACCESS_READ)])                                # 1
    prog.task(L.BODY_NOP, [(0, L.ACCESS_READ)])                                      # 2
    prog.task(L.BODY_CHECK_I32, [(0, L.ACCESS_READ)])                                # 3
    prog.task(L.BODY_CHECK_F32, [(0, L.ACCESS_READ)])                                # 4
    prog.task(L.BODY_FILL_I32, [(1, L.ACCESS_WRITE), (3, L.ACCESS_READ)])             # 5: wider tile 3
    prog.task(L.BODY_CHECK_I32, [(1, L.ACCESS_READ)])
    prog.task(L.BODY_CHECK_I32, [(1, L.ACCESS_READ)])
    prog.task(L.BODY_COPY, [(2, L.ACCESS_READ), (1, L.ACCESS_RW)])                    # 8: unequal sizes
    prog.task(L.BODY_CHECK_I32, [(1, L.ACCESS_READ)])
    prog.task(L.BODY_CHECK_I32, [(1, L.ACCESS_READ)])
    prog.task(L.BODY_INCR_I32, [(1, L.ACCESS_RW | L.FLOW_PUSHOUT)])                   # 11: pushout of X
    prog.task(L.BODY_CHECK_I32, [(1, L.ACCESS_READ)])
    prog.task(L.BODY_CHECK_I32, [(1, L.ACCESS_READ)])
    prog.task(L.BODY_COPY, [(1, L.ACCESS_READ), (0, L.ACCESS_WRITE)])                 # 14: fuses with the first 8 of 10
    for _ in range(10):
        prog.task(L.BODY_CHECK_I32, [(0, L.ACCESS_READ)])
    groups, fused = R.read_groups(prog.dag(), nbytes)
    assert fused == {0: [3, 4], 14: list(range(15, 23))}
    assert groups == {3: [3, 4], 6: [6, 7], 9: [9, 10], 12: [12, 13], 15: list(range(15, 23)), 23: [23, 24]}
    assert R.read_groups(prog.dag(), nbytes, fuse=False)[1] == {}


@pytest.mark.parametrize("seed", range(2))
def test_gemm_chains_beside_every_body_match_the_oracle(seed):
    prog, layout = random_case(seed, ntasks=200)
    prog = R.program(prog)
    copy_to = next(fl[0][0] for b, fl, *_ in prog.tasks if b == L.BODY_IOTA_I32)      # an int tile
    prog, layout = R.with_gemm_chains(np.random.default_rng(seed), prog, layout, copy_to)
    ref = same_as_oracle(prog, layout)
    gemms = [t for t, (b, *_) in enumerate(prog.tasks) if b == L.BODY_GEMM_BF16]
    assert len(gemms) == sum(c[3] for c in R.GEMM_CHAINS)
    # the GEMMs changed their C tiles, and the COPY out of the first one reached the int tile
    assert ref["stats"]["bytes_d2h"] > 0 and any(ref["result"][gemms[-1] + 1:] >> 32)


def test_inexact_gemm_data_trips_the_reference():
    M, N, K = 2, 8, 8
    a, b, c = np.ones((M, K), np.float32), np.ones((N, K), np.float32), np.zeros((M, N), np.float32)
    bits = lambda x: f32_to_bf16_bits(x).reshape(-1).view(np.uint8).copy()
    R.run_body(L.BODY_GEMM_BF16, [bits(a), bits(b), bits(c)], (M, N, K))
    flows = [bits(a), bits(b), np.concatenate([bits(c), np.full(6, 7, np.uint8)])]
    R.run_body(L.BODY_GEMM_BF16, flows, (M, N, K))
    assert np.all(bf16_bits_to_f32(flows[2][:M * N * 2].view(np.uint16)) == K) and np.all(flows[2][M * N * 2:] == 7)
    for a2, c2 in ((a * 0.5, c), (a, c + 250), (a * 40, c)):         # a fraction; past 256; a partial sum past 256
        with pytest.raises(AssertionError, match="exact regime"):
            R.run_body(L.BODY_GEMM_BF16, [bits(a2), bits(b), bits(c2)], (M, N, K))
