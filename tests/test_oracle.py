"""Pins the CPU oracle (oracle/) against the reference: known answers of the reference's own tests and
examples, and the reference's own compiled code -- live where oracle/_ref was built from the reference's sources,
replayed from its recorded answers (tests/golden/reference_pieces.json.gz) everywhere else.
No GPU needed."""
import ctypes as C
import gzip
import json
import os
import random

import numpy as np
import pytest

from oracle import orc, orc_dags as dags

HAVE_REF_ZONE = os.path.exists(orc.REF_ZONE_PATH)
HAVE_REF_DATA = os.path.exists(orc.REF_DATA_PATH)
HAVE_REF_TWODBC = os.path.exists(orc.REF_TWODBC_PATH)
HAVE_REF_SELECT = os.path.exists(orc.REF_SELECT_PATH)
GOLDEN_PIECES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pieces.json.gz")
RECORDED = {}           # piece -> answers of the live library, in call order (tests/golden/make_golden.py writes them out)
_VOID = {"ref_twodbc_free", "ref_sel_init", "ref_sel_set_load", "zone_free", "ref_data_add_copy", "ref_data_set", "ref_end_transfer"}


def _is_out(a):
    return isinstance(a, C.Array) or type(a).__name__ == "CArgObject"


class Reference:
    """One piece of the reference compiled from its own sources (oracle/Makefile.ref), seen through its answers in call
    order: return values and out-parameters (ctypes arrays, byref).  With the library (`lib`) the calls go to it and are
    recorded; without it they are replayed from the golden file, so the oracle is held to the same answers.  zone_malloc
    answers are kept relative to `base`, the arena the test hands the allocator."""

    def __init__(self, piece, lib, base=0):
        self.piece, self.lib, self.base = piece, lib, base
        if lib is not None:
            self.log = RECORDED.setdefault(piece, [])
            del self.log[:]
        else:
            with gzip.open(GOLDEN_PIECES, "rt") as f:
                self.log = json.load(f)[piece][::-1]

    def __getattr__(self, fn):
        def call(*args):
            outs = [a._obj if type(a).__name__ == "CArgObject" else a for a in args if _is_out(a)]
            if self.lib is not None:
                r = getattr(self.lib, fn)(*args)
                if fn not in _VOID:
                    rec = (-1 if not r else r - self.base) if fn == "zone_malloc" else r
                    self.log.append([fn, rec] + [list(o) if isinstance(o, C.Array) else o.value for o in outs])
                return r
            if fn in _VOID:
                return None
            e = self.log.pop()
            assert e[0] == fn, ("replay out of step", e[0], fn)
            for o, v in zip(outs, e[2:]):
                if isinstance(o, C.Array):
                    o[:] = v
                else:
                    o.value = v
            if fn == "zone_malloc":
                return None if e[1] < 0 else self.base + e[1]
            return e[1]
        return call


def tiles_for(dag, valid=False):
    t = np.zeros(dag.ntiles, orc.TILE_DTYPE)
    t["bytes"] = dag.tile_bytes
    t["src_ptr"] = np.arange(dag.ntiles, dtype=np.uint64) * np.uint64(dag.tile_bytes)   # offsets into host
    t["state"] = orc.TILE_VALID if valid else orc.TILE_INVALID
    return t


# ------------------------------------------------------------------ DAG execution known answers
@pytest.mark.parametrize("NB", [0, 1, 10, 999])
def test_ex02_chain_known_answer(NB):
    """Ex02_Chain.jdf:44-50: 'I am element k in the chain' -- task k observes k, final value NB (config 1)."""
    dag = dags.ex02_chain(NB)
    out = orc.run_window(dag.tasks, dag.succ, tiles_for(dag), dag.ready, np.zeros(1, np.int32))
    assert out["rc"] == 0 and out["stats"]["tasks_retired"] == NB + 1
    assert np.array_equal(out["retire_order"], np.arange(NB + 1))
    assert np.array_equal(out["seen_version"][:, 0], np.arange(NB + 1))
    assert out["device"][0].view(np.int32)[0] == NB
    assert out["stats"]["bytes_h2d"] == 0                  # NEW data is never pulled in (device_gpu.c:2049)


@pytest.mark.parametrize("K,NB", [(1, 0), (4, 6), (37, 14)])
def test_ex05_broadcast_known_answer(K, NB):
    """Ex05_Broadcast.jdf:33-39,53-57: every TaskRecv(k, n) prints k."""
    dag = dags.ex05_broadcast(K, NB, 64)
    host = np.full(K * 16, -1, np.int32)
    out = orc.run_window(dag.tasks, dag.succ, tiles_for(dag), dag.ready, host)
    F = NB // 2 + 1
    assert out["rc"] == 0 and out["stats"]["body_errors"] == 0
    assert np.array_equal(out["result"][K:] & np.uint64(0xFFFFFFFF), np.repeat(np.arange(K), F).astype(np.uint64))
    assert out["stats"]["bytes_h2d"] == K * 64 and out["stats"]["stage_ins"] == K


@pytest.mark.parametrize("NB_TOKEN", [1, 3, 16])
def test_ptg_pingpong_known_answer(NB_TOKEN):
    """ptg_pingpong.jdf:144-149: after INIT(i) + CPU(+i) + GPU(+i) every element is 3*i."""
    dag = dags.ptg_pingpong(NB_TOKEN)
    host = np.zeros(2 * NB_TOKEN, np.int32)
    out = orc.run_window(dag.tasks, dag.succ, tiles_for(dag), dag.ready, host)
    assert out["rc"] == 0
    assert np.array_equal(host, 3 * np.arange(2 * NB_TOKEN))


def test_dtd_new_tile_known_answer():
    """dtd_test_new_tile_cuda_kernels.cu:17,30,47-49: init i, times two => 2*i, and the accumulated sum."""
    dag = dags.dtd_new_tile(5, 100)
    out = orc.run_window(dag.tasks, dag.succ, tiles_for(dag), dag.ready, np.zeros(500, np.int32))
    assert out["rc"] == 0
    for d in out["device"]:
        assert np.array_equal(d.view(np.int32), 2 * np.arange(100))
    assert sum(int(d.view(np.int32).sum()) for d in out["device"]) == 5 * 2 * (99 * 100 // 2)


def test_rtt_chain_known_answer():
    """rtt.jdf:26-47 with body T += 1: after NT hops T == T0 + NT; the last hop writes back to A(f, k%WS)."""
    dag = dags.rtt_chain(17, 3, 64)
    host = np.arange(48, dtype=np.float32)
    expect = host + 17
    out = orc.run_window(dag.tasks, dag.succ, tiles_for(dag), dag.ready, host)
    assert out["rc"] == 0 and np.array_equal(host, expect)
    assert np.all(out["tiles"]["version"] == 17)


def test_deadlock_is_reported():
    dag = dags.ex02_chain(4)
    dag.tasks["dep_goal"][2] = 0x3
    out = orc.run_window(dag.tasks, dag.succ, tiles_for(dag), dag.ready, np.zeros(1, np.int32))
    assert out["rc"] == -1 and out["stats"]["tasks_retired"] == 2


def test_gemm_body_matches_numpy():
    from parsec_b200.bf16 import bf16_bits_to_f32, f32_to_bf16_bits, round_to_bf16
    rng = np.random.default_rng(3)
    T, NT = 32, 2
    A, B, Cm = (round_to_bf16(rng.uniform(-.5, .5, (NT, NT, T, T)).astype(np.float32)) for _ in range(3))
    dag = dags.dtd_gemm(NT, T)
    host = np.concatenate([f32_to_bf16_bits(x).ravel() for x in (A, B, Cm)])
    out = orc.run_window(dag.tasks, dag.succ, tiles_for(dag), dag.ready, host)
    assert out["rc"] == 0
    got = bf16_bits_to_f32(host[2 * NT * NT * T * T:]).reshape(NT, NT, T, T)
    for i in range(NT):
        for j in range(NT):
            c = Cm[i, j].copy()
            for k in range(NT):
                c = round_to_bf16(c + A[i, k] @ B[k, j].T)
            assert np.allclose(got[i, j], c, rtol=2 ** -7, atol=2 ** -7)


# ------------------------------------------------------------------ DTD ordering rule
def test_dtd_rule_gemm_matches_builder():
    """The per-tile last-writer / readers rule applied to dtd_test_simple_gemm.c:675-696's insertion order
    gives exactly the C(i,j) chains of the numpy builder."""
    NT = 4
    dag = dags.dtd_gemm(NT)
    n = dag.ntasks
    nbf = np.full(n, 3, np.int32)
    ft = np.full((n, 4), -1, np.int32)
    ft[:, :3] = dag.tasks["tile"][:, :3]
    fo = np.zeros((n, 4), np.int32)
    fo[:, 0] = fo[:, 1] = orc.DTD_INPUT
    fo[:, 2] = orc.DTD_INOUT
    src, dst, fl, dep = orc.dtd_build(nbf, ft, fo, dag.ntiles)
    es, ed, ef = dag.edges()
    assert sorted(zip(src.tolist(), dst.tolist(), fl.tolist())) == sorted(zip(es.tolist(), ed.tolist(), ef.tolist()))
    assert np.array_equal(dep, dag.tasks["dep_goal"])


def test_dtd_rule_war_and_reader_runs():
    """W0 R1 R2 R3 W4 R5 on one tile: readers wait for W0 only; W4 waits for W0 and R1..R3 (WAR gate,
    insert_function.c:2102-2118); R5 waits for W4."""
    ops = [orc.DTD_INOUT, orc.DTD_INPUT, orc.DTD_INPUT, orc.DTD_INPUT, orc.DTD_INOUT, orc.DTD_INPUT]
    n = len(ops)
    ft = np.full((n, 4), -1, np.int32); ft[:, 0] = 0
    fo = np.zeros((n, 4), np.int32); fo[:, 0] = ops
    src, dst, fl, dep = orc.dtd_build(np.ones(n, np.int32), ft, fo, 1)
    edges = sorted(zip(src.tolist(), dst.tolist()))
    assert edges == [(0, 1), (0, 2), (0, 3), (0, 4), (1, 4), (2, 4), (3, 4), (4, 5)]
    assert dep.tolist() == [0, 1, 1, 1, 4, 1]


# ------------------------------------------------------------------ 2D block cyclic map
@pytest.mark.parametrize("P,Q,kp,kq,ip,jq", [(1, 1, 1, 1, 0, 0), (2, 2, 1, 1, 0, 0), (2, 4, 1, 1, 1, 3), (1, 4, 1, 1, 0, 0),
                                              (2, 3, 2, 3, 0, 0), (3, 2, 2, 2, 1, 1)])
def test_twodbc_owner_and_slots(P, Q, kp, kq, ip, jq):
    """two_dim_rectangle_cyclic.c:258-286, 351-412: every tile has exactly one owner, the owner's local slots
    are a bijection onto [0, nb_local_tiles), key = n*lmt + m round-trips (key2coords)."""
    L = orc.lib()
    mb = nb = 4
    lm, ln = 4 * 11, 4 * 7
    ds = [orc.twodbc(r, mb, nb, lm, ln, P=P, Q=Q, kp=kp, kq=kq, ip=ip, jq=jq) for r in range(P * Q)]
    total = 0
    for r, d in enumerate(ds):
        slots = set()
        for m in range(d.mt):
            for n in range(d.nt):
                owner = L.orc_twodbc_rank_of(C.byref(d), m, n)
                pos = L.orc_twodbc_position(C.byref(d), m, n)
                assert (pos >= 0) == (owner == r)
                if owner == r:
                    assert pos not in slots and 0 <= pos < d.nb_local_tiles
                    slots.add(pos)
                    assert L.orc_twodbc_tile_offset_elems(C.byref(d), m, n) == pos * mb * nb
                key = L.orc_twodbc_key(C.byref(d), m, n)
                assert key == n * d.lmt + m
                mm, nn = C.c_int(), C.c_int()
                L.orc_twodbc_key2coords(C.byref(d), key, C.byref(mm), C.byref(nn))
                assert (mm.value, nn.value) == (m, n)
        assert len(slots) == d.nb_local_tiles
        total += len(slots)
    assert total == ds[0].mt * ds[0].nt
    if kp == kq == 1 and ip == jq == 0:
        d = ds[0]
        for m in range(d.mt):
            for n in range(d.nt):
                assert L.orc_twodbc_rank_of(C.byref(d), m, n) == (m % P) * Q + (n % Q)   # SURVEY 8(e)


def test_twodbc_oracle_and_product_equal_reference_build():
    """The reference's own two_dim_rectangle_cyclic.c (compiled from the reference's sources) vs the oracle's restatement
    vs the product's pb2_matrix_block_cyclic_new: owner, key, derived sizes, for plain, k-cyclic and offset grids, full
    and sub-matrices, every rank."""
    from parsec_b200 import runtime as R
    ref = Reference("twodbc", orc.ref_twodbc() if HAVE_REF_TWODBC else None)
    L = orc.lib()
    rl = R.lib()
    rng = random.Random(2026)
    ctxp = C.c_void_p()
    assert rl.pb2_init(C.byref(ctxp), 1) == 0
    try:
        for case in range(60):
            P, Q = rng.choice([(1, 1), (1, 4), (2, 2), (2, 4), (3, 2), (4, 1)])
            kp, kq = rng.choice([(1, 1), (1, 1), (2, 1), (2, 3), (3, 2)])
            ip, jq = rng.randrange(P), rng.randrange(Q)
            mb, nb = rng.choice([(4, 4), (3, 5), (8, 2)])
            lm, ln = mb * rng.randrange(3, 14) + rng.randrange(mb), nb * rng.randrange(3, 12) + rng.randrange(nb)
            i, j = (0, 0) if case % 3 else (rng.randrange(lm // 2), rng.randrange(ln // 2))
            m, n = lm - i - rng.randrange(0, (lm - i) // 3 + 1), ln - j - rng.randrange(0, (ln - j) // 3 + 1)
            for rank in range(P * Q):
                args = (rank, mb, nb, lm, ln, i, j, m, n, P, Q, kp, kq, ip, jq)
                rd = ref.ref_twodbc_new(*args)
                od = orc.twodbc(rank, mb, nb, lm, ln, i, j, m, n, P, Q, kp, kq, ip, jq)
                pd = C.c_void_p(rl.pb2_matrix_block_cyclic_new(ctxp, 4, *args))
                assert pd.value
                info = (C.c_int64 * 12)()
                ref.ref_twodbc_info(rd, info)
                assert (od.lmt, od.lnt, od.mt, od.nt, od.nb_elem_r, od.nb_elem_c, od.nb_local_tiles, od.bsiz, od.llm, od.lln,
                        od.rrank, od.crank) == tuple(info), (case, args)
                pinfo = (C.c_int64 * 8)()
                assert rl.pb2_dc_info(pd, pinfo) == 0
                assert tuple(pinfo)[:7] == tuple(info)[:7], (case, args)
                for mm in range(od.mt):
                    for nn in range(od.nt):
                        r_ref = ref.ref_twodbc_rank_of(rd, mm, nn)
                        assert L.orc_twodbc_rank_of(C.byref(od), mm, nn) == r_ref, (case, args, mm, nn)
                        assert rl.pb2_dc_rank_of(pd, mm, nn) == r_ref, (case, args, mm, nn)
                        k_ref = ref.ref_twodbc_key(rd, mm, nn)
                        assert L.orc_twodbc_key(C.byref(od), mm, nn) == k_ref == rl.pb2_dc_data_key(pd, mm, nn)
                        assert ref.ref_twodbc_rank_of_key(rd, k_ref) == r_ref
                rl.pb2_data_collection_free(pd)
                ref.ref_twodbc_free(rd)
    finally:
        rl.pb2_fini(C.byref(ctxp))


def test_twodbc_rtt_placement():
    """rtt_main.c:191-198 / rtt.jdf:30: PING(k, f) lives on A(f, k % WS) of a 1 x WS grid => owner k % WS."""
    WS, FRAGS = 4, 3
    d = orc.twodbc(0, 8, 8, 8 * FRAGS, 8 * WS, P=1, Q=WS)
    for k in range(20):
        for f in range(FRAGS):
            assert orc.lib().orc_twodbc_rank_of(C.byref(d), f, k % WS) == k % WS


# ------------------------------------------------------------------ LCG generator
def test_lcg_jump_equals_stepping():
    """dtd_test_simple_gemm.c:154-172: Rnd64_jump(n, seed) is n steps of x <- A*x + C."""
    L = orc.lib()
    for seed in (1789, 1805, 1901):
        x = seed
        for n in range(0, 70):
            assert L.orc_rnd64_jump(n, seed) == x
            x = L.orc_rnd64_step(x)
        assert L.orc_rnd64_jump(12345 + 678, seed) == L.orc_rnd64_jump(678, L.orc_rnd64_jump(12345, seed))


def test_lcg_tile_is_a_window_of_the_global_matrix():
    """A tile generated at (m, n) equals the same window of the matrix generated as one tile (jump-ahead)."""
    L = orc.lib()
    M, mb = 24, 8
    full = np.zeros((M, M), np.float32, order="F")
    L.orc_lcg_tile(full.ctypes.data_as(C.c_void_p), 0, 0, M, M, M, M, 1789)
    t = np.zeros((mb, mb), np.float32, order="F")
    L.orc_lcg_tile(t.ctypes.data_as(C.c_void_p), 8, 16, mb, mb, M, mb, 1789)
    assert np.array_equal(t, full[8:16, 16:24])
    assert np.all(np.abs(full) <= 0.5)


# ------------------------------------------------------------------ device selection
def _sel(devs, access, present, pref, owner, skew=20, allow_cpu=0):
    arr = (orc.SelDev * len(devs))(*[orc.SelDev(*d) for d in devs])
    a = [np.array(x, np.int32) for x in (access, present, pref, owner)]
    return orc.lib().orc_select_best_device(arr, len(devs), len(access), *[x.ctypes.data_as(C.c_void_p) for x in a], skew, allow_cpu)


def test_select_oracle_equals_reference_build():
    """The reference's own parsec_select_best_device (device.c:100-310, compiled from its sources, driven with fake
    device modules and tasks) vs the oracle: 4000 random tasks over a CPU, the recursive device and four GPUs --
    affinity by preferred/owner device, ETA with the 20 % skew, taskpool device masks, CPU incarnations with and
    without load_balance_allow_cpu."""
    ref = Reference("select", orc.ref_select() if HAVE_REF_SELECT else None)
    CPU, REC, CUDA = 1, 2, 4
    types = [CPU, REC, CUDA, CUDA, CUDA, CUDA]
    rng = random.Random(77)
    ref.ref_sel_init(20, 0)
    for t in types:
        assert ref.ref_sel_add_device(t, 0, 1) >= 0
    for allow_cpu in (0, 1):
        for skew in (20, 0, 50):
            ref.ref_sel_init(skew, allow_cpu)
            for case in range(700):
                loads = [rng.choice([0, 0, rng.randrange(0, 5000)]) for _ in types]
                ests = [rng.randrange(1, 400) for _ in types]
                for d in range(len(types)):
                    ref.ref_sel_set_load(d, loads[d], ests[d])
                nb = rng.randrange(1, 5)
                access = [rng.choice([0x04, 0x08, 0x0C]) for _ in range(nb)]
                present = [rng.choice([1, 1, 1, 0]) for _ in range(nb)]
                pref = [rng.choice([-1, -1, -1, 0, 2, 3, 4, 5]) for _ in range(nb)]
                owner = [rng.choice([-1, 0, 0, 2, 3, 4, 5]) for _ in range(nb)]
                chore = CUDA | (CPU if rng.random() < 0.4 else 0)
                mask = rng.choice([0x3f, 0x3f, 0x3d, 0x0f, 0x35, 0x31, 0x03])
                a = [np.array(x, np.int32) for x in (access, present, pref, owner)]
                load = C.c_int64()
                got = ref.ref_sel_select(nb, *[x.ctypes.data_as(C.c_void_p) for x in a], chore, mask, C.byref(load))
                devs = [(1 if types[d] == CUDA else 0, 1 if types[d] == REC else 0,
                         1 if ((mask >> d) & 1) and (types[d] & chore) else 0, loads[d], ests[d]) for d in range(len(types))]
                want = _sel(devs, access, present, pref, owner, skew, allow_cpu)
                assert got == want, (case, allow_cpu, skew, devs, access, present, pref, owner, chore, hex(mask))
                if got >= 0:
                    assert load.value == ests[got]


def test_select_best_device_rules():
    # devices: 0 cpu, 1 recursive, 2..5 gpus; (is_gpu, is_recursive, enabled, load, estimate)
    devs = [(0, 0, 1, 0, 10), (0, 1, 1, 0, 10), (1, 0, 1, 0, 10), (1, 0, 1, 0, 10), (1, 0, 1, 0, 10), (1, 0, 1, 0, 10)]
    RW, R = 0x0C, 0x04
    # get_best_device_check.jdf:68-83: preferred_device of the written tile decides: gpu (n*nt+m) % ngpu
    nt, ngpu = 5, 4
    for m in range(nt):
        for n in range(nt):
            g = 2 + (n * nt + m) % ngpu
            assert _sel(devs, [RW], [1], [g], [0]) == g
    assert _sel(devs, [RW, R], [1, 1], [-1, -1], [3, 4]) == 3           # written data already on gpu 3
    assert _sel(devs, [R, RW], [1, 1], [-1, -1], [4, 0]) == 4           # read data on gpu 4 -> rdata_dev, idle
    assert _sel(devs, [R], [1], [-1], [0]) == 5                          # no affinity: least ETA, highest index first
    loaded = [list(d) for d in devs]
    loaded[4][3] = 100                                                   # gpu 4 busy: (100+10)/1.2 > 10 => move
    assert _sel(loaded, [R], [1], [-1], [4]) == 5
    loaded[4][3] = 1                                                     # (1+10)/1.2 < 10 => stay (20 % skew)
    assert _sel(loaded, [R], [1], [-1], [4]) == 4
    only_cpu = [(0, 0, 1, 0, 10)] + [(1, 0, 0, 0, 10)] * 3
    assert _sel(only_cpu, [R], [1], [-1], [0]) == 0
    assert _sel([(0, 0, 0, 0, 1)], [R], [1], [-1], [0]) == -1


# ------------------------------------------------------------------ zone allocator
def _zone_scenario(zm, zf):
    """tests/runtime/cuda/zonemalloc.c:32-80 (128 segments of 512 B)."""
    N = 128
    seg = [zm(512) for _ in range(N)]
    assert all(s is not None for s in seg) and sorted(seg) == list(range(N))
    assert zm(512) is None
    for s in seg: zf(s)
    seg = [zm(512) for _ in range(N)]
    assert all(s is not None for s in seg)
    for i in range(0, N, 2): zf(seg[i])
    for i in range(1, N, 2): zf(seg[i])
    seg = [zm(512 // ((i % 2) + 1)) for i in range(N)]
    assert all(s is not None for s in seg)
    for i in range(N - 1, 0, -1): zf(seg[i])
    return seg[0]


def test_zone_reference_scenario():
    L = orc.lib()
    z = L.orc_zone_init(128, 512)
    def zm(sz):
        r = L.orc_zone_malloc(z, sz)
        return None if r < 0 else r
    first = _zone_scenario(zm, lambda s: L.orc_zone_free(z, s))
    assert L.orc_zone_in_use(z) == 512
    assert L.orc_zone_free(z, first) == 0 and L.orc_zone_free(z, first) == -2    # double free is reported
    nfree, largest = C.c_int(), C.c_int()
    L.orc_zone_free_profile(z, C.byref(nfree), C.byref(largest))
    assert (nfree.value, largest.value) == (1, 128)                              # fully coalesced again
    assert L.orc_zone_malloc(z, 0) == -1
    L.orc_zone_fini(z)


def test_zone_oracle_equals_reference_build():
    """Same malloc/free sequences through the REAL parsec/utils/zone_malloc.c (compiled by oracle/Makefile.ref)
    and through the restatement: identical addresses and in-use bytes at every step."""
    lib = C.CDLL(orc.REF_ZONE_PATH) if HAVE_REF_ZONE else None
    L = orc.lib()
    if lib is not None:
        lib.zone_malloc_init.restype = C.c_void_p; lib.zone_malloc_init.argtypes = [C.c_void_p, C.c_int, C.c_size_t]
        lib.zone_malloc.restype = C.c_void_p; lib.zone_malloc.argtypes = [C.c_void_p, C.c_size_t]
        lib.zone_free.argtypes = [C.c_void_p, C.c_void_p]
        lib.zone_in_use.restype = C.c_size_t; lib.zone_in_use.argtypes = [C.c_void_p]
    NSEG, UNIT = 96, 512
    buf = (C.c_char * (NSEG * UNIT))()
    base = C.addressof(buf)
    ref = Reference("zone", lib, base)
    for seed in range(25):
        rnd = random.Random(seed)
        zr, zo = ref.zone_malloc_init(base, NSEG, UNIT), L.orc_zone_init(NSEG, UNIT)
        live = []
        for _ in range(1500):
            if live and rnd.random() < 0.45:
                tid = live.pop(rnd.randrange(len(live)))
                ref.zone_free(zr, base + tid * UNIT)
                assert L.orc_zone_free(zo, tid) == 0
            else:
                size = rnd.choice([1, 256, 512, 513, 1024, 2000, 4096, 8192])
                pr, to = ref.zone_malloc(zr, size), L.orc_zone_malloc(zo, size)
                assert (-1 if not pr else (pr - base) // UNIT) == to
                if to >= 0: live.append(to)
            assert ref.zone_in_use(zr) == L.orc_zone_in_use(zo)
        L.orc_zone_fini(zo)


# ------------------------------------------------------------------ coherency protocol
def test_coherency_oracle_equals_reference_build():
    """Random start/end_transfer_ownership sequences through the REAL parsec/data.c (compiled by
    oracle/Makefile.ref) and the restatement leave identical host-visible state and return values."""
    lib = C.CDLL(orc.REF_DATA_PATH) if HAVE_REF_DATA else None
    L = orc.lib()
    if lib is not None:
        lib.ref_data_new.restype = C.c_void_p
        for fn in (lib.ref_data_add_copy, lib.ref_data_set, lib.ref_data_get, lib.ref_data_owner, lib.ref_start_transfer,
                   lib.ref_end_transfer, lib.ref_data_set_owner):
            fn.argtypes = None
    ref = Reference("data", lib)
    NDEV = 6
    assert ref.ref_data_setup(NDEV) == 0
    R, W = 0x04, 0x08
    for seed in range(200):
        rnd = random.Random(seed)
        rd = C.c_void_p(ref.ref_data_new())
        od = orc.OrcData()
        L.orc_data_create(C.byref(od), NDEV, 0)
        writer_legal = True
        for step in range(12):
            dev = rnd.randrange(2, NDEV)
            acc = rnd.choice([R, W, R | W, R, R | W])
            if not od.copy[dev].present:
                ref.ref_data_add_copy(rd, dev)
                od.copy[dev].present = 1
            # a sane program never has two owners: skip accesses the reference asserts against
            if od.copy[dev].coherency_state == 0x1 and od.owner_device != dev:
                continue
            r_ref = ref.ref_start_transfer(rd, dev, acc)
            r_orc = L.orc_data_start_transfer_ownership(C.byref(od), dev, acc)
            assert r_ref == r_orc, (seed, step, dev, acc)
            ref.ref_end_transfer(rd, dev, acc)
            L.orc_data_end_transfer_ownership(C.byref(od), dev, acc)
            if acc & W:   # what stage_in does next: the written replica gets a newer version
                src = r_orc if r_orc >= 0 else dev
                v = od.copy[src].version + 1
                od.copy[dev].version = v
                out = (C.c_int * 5)()
                ref.ref_data_get(rd, dev, out)
                ref.ref_data_set(rd, dev, out[1], out[2], v, out[3])
            elif r_orc >= 0:
                v = od.copy[r_orc].version
                od.copy[dev].version = v
                out = (C.c_int * 5)()
                ref.ref_data_get(rd, dev, out)
                ref.ref_data_set(rd, dev, out[1], out[2], v, out[3])
            assert ref.ref_data_owner(rd) == od.owner_device
            for d in range(NDEV):
                out = (C.c_int * 5)()
                ref.ref_data_get(rd, d, out)
                assert out[0] == od.copy[d].present
                if out[0]:
                    assert (out[1], out[3], out[4]) == (od.copy[d].coherency_state, od.copy[d].readers, od.copy[d].version), (seed, step, d)


def test_gpu_task_protocol_versions():
    """RW on a GPU: H2D from the host, version+1, OWNED; a second GPU reading the same version pulls D2D from the
    first (device_gpu.c:1892-2008); pushout brings the host copy to the GPU's version (device_gpu.c:3247-3255)."""
    L = orc.lib()
    R, W = 0x04, 0x08
    d = orc.OrcData()
    L.orc_data_create(C.byref(d), 4, 0)
    req = C.c_int()
    peer = 0b1100
    assert L.orc_gpu_stage_in(C.byref(d), 2, 0, R | W, peer, C.byref(req)) == 0       # H2D from the host
    assert d.copy[2].version == 1 and d.copy[2].data_transfer_status == 1
    L.orc_gpu_stage_in_complete(C.byref(d), 2, R | W)
    assert d.copy[2].coherency_state == 0x1 and d.owner_device == 2 and d.copy[0].coherency_state == 0x4
    L.orc_gpu_task_complete(C.byref(d), 2, R | W, 0)
    assert d.copy[2].readers == 0
    # successor on GPU 3 reads the GPU-2 replica (its data_in): D2D
    assert L.orc_gpu_stage_in(C.byref(d), 3, 2, R, peer, C.byref(req)) == 2
    assert d.copy[3].version == 1
    L.orc_gpu_stage_in_complete(C.byref(d), 3, R)
    assert d.copy[3].coherency_state == 0x4
    L.orc_gpu_task_complete(C.byref(d), 3, R, 0)
    # another RW on GPU 2 with pushout: already there, version 2, host follows
    assert L.orc_gpu_stage_in(C.byref(d), 2, 2, R | W, peer, C.byref(req)) == -1
    assert d.copy[2].version == 2
    L.orc_gpu_task_complete(C.byref(d), 2, R | W, 1)
    assert d.copy[0].version == 2 and d.copy[0].coherency_state == 0x4 and d.copy[2].coherency_state == 0x4
    # NEW data is never transferred
    n = orc.OrcData()
    L.orc_data_create(C.byref(n), 4, 1)
    assert L.orc_gpu_stage_in(C.byref(n), 2, 0, R | W, peer, C.byref(req)) == -1
    assert n.copy[2].version == 1 and n.copy[2].data_transfer_status == 2


# ------------------------------------------------------------------ CPU scheduler port == sequential oracle
@pytest.mark.parametrize("nthreads", [1, 4])
def test_cpu_scheduler_port_results(nthreads):
    dag = dags.ex05_broadcast(64, 14, 256)
    host = np.zeros(64 * 64, np.int32)
    t = tiles_for(dag, valid=True)
    t["dev_ptr"] = host.ctypes.data + np.arange(64, dtype=np.uint64) * np.uint64(256)
    secs, per_thread, errs = orc.cpu_sched_run(dag.tasks, dag.succ, t, dag.ready, nthreads)
    assert secs > 0 and errs == 0 and per_thread.sum() == dag.ntasks
    assert np.array_equal(host.reshape(64, 64)[:, 0], np.arange(64))
