"""Sharding a task pool over the GPUs of one box: one process per GPU, 2D block-cyclic owner map, NCCL over
NVLink for the dependency edges that cross GPUs.

The reference spreads a PTG over processes with the collection's rank_of (two_dim_rectangle_cyclic.c:258-286):
a task runs where its affinity datum lives; an edge whose endpoints have different owners is a remote
dependency (remote_dep.c): ACTIVATE message, then the tile itself (remote_dep_mpi.c:1681, :2120).  Here the
same split is computed on the host of every rank, the local parts run as device windows, and all the tiles a
window produced for remote successors travel in one NCCL exchange (send/recv pairs over NVLink) before the
window that consumes them -- the ACTIVATE/GET/PUT hand-shake of a whole dependency frontier batched into one
collective step, no per-edge host round trip.

Two data paths are kept:
  * "direct" (default): ONE window per GPU for the whole pool; an edge that crosses GPUs is released by the producer's
    worker CTA with a system-scope atomic on the consumer GPU's dependency word plus a ring write over NVLink
    (release_remote_warp), and the consumer's worker pulls the tile out of the producer's slab when the task runs
    (stage_in_flow, src_kind PEER).  No host and no collective on the data path; NCCL is only the per-step
    barrier that orders "every rank has reset its window" before "any rank starts".
  * "exchange": two windows per GPU with one batched NCCL send/recv of the frontier in between (kept as the
    library baseline the direct path is measured against).

Host logic only (numpy + torch.distributed plumbing); the kernels are the engine's.
"""
import ctypes as C
import os

import numpy as np

from . import _lib as L


class Partition:
    """pb2_partition_* (include/pb2_engine.h): split a dependency-closed window over `nranks` GPUs."""

    def __init__(self, tasks, succ, tiles, ready, task_rank, tile_rank, nranks, part_bytes=0):
        self._lib = L.load()
        self._h = C.c_void_p()
        tasks = np.ascontiguousarray(tasks, L.TASK_DTYPE)
        succ = np.ascontiguousarray(succ, np.uint32)
        tiles = np.ascontiguousarray(tiles, L.TILE_DTYPE)
        ready = np.ascontiguousarray(ready, np.int32)
        task_rank = np.ascontiguousarray(task_rank, np.int32)
        tile_rank = np.ascontiguousarray(tile_rank, np.int32)
        assert len(task_rank) == len(tasks) and len(tile_rank) == len(tiles)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        rc = self._lib.pb2_partition_create(C.byref(self._h), vp(tasks), len(tasks), vp(succ), len(succ), vp(tiles), len(tiles),
                                            vp(ready), len(ready), vp(task_rank), vp(tile_rank), nranks, part_bytes)
        if rc != L.PB2_SUCCESS:
            raise L.Pb2Error(rc, "pb2_partition_create", (self._lib.pb2_partition_error() or b"").decode())
        self.nranks = nranks

    def sizes(self, rank):
        s = L.PartitionSizes()
        rc = self._lib.pb2_partition_sizes(self._h, rank, C.byref(s))
        if rc != L.PB2_SUCCESS:
            raise L.Pb2Error(rc, "pb2_partition_sizes", "")
        return {f[0]: getattr(s, f[0]) for f in L.PartitionSizes._fields_}

    def get(self, rank, slab_base):
        """slab_base[r] = address of rank r's slab as seen from `rank`."""
        z = self.sizes(rank)
        out = {
            "tasks": np.zeros(z["ntasks"], L.TASK_DTYPE), "succ": np.zeros(z["nsucc"], np.uint32),
            "tiles": np.zeros(z["ntiles"], L.TILE_DTYPE), "ready": np.zeros(z["nready"], np.int32),
            "rs_begin": np.zeros(z["ntasks"] + 1, np.int32), "rs_rank": np.zeros(z["nremote"], np.int32),
            "rs_target": np.zeros(z["nremote"], np.uint32), "global_id": np.zeros(z["ntasks"], np.int32),
            "slot_tile": np.zeros(z["nslots"], np.int32), "slot_offset": np.zeros(z["nslots"], np.uint64),
        }
        base = np.ascontiguousarray(slab_base, np.uint64)
        assert len(base) == self.nranks
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        rc = self._lib.pb2_partition_get(self._h, rank, vp(base), *[vp(out[k]) for k in (
            "tasks", "succ", "tiles", "ready", "rs_begin", "rs_rank", "rs_target", "global_id", "slot_tile", "slot_offset")])
        if rc != L.PB2_SUCCESS:
            raise L.Pb2Error(rc, "pb2_partition_get", "")
        out["slab_bytes"] = z["slab_bytes"]
        return out

    def set_push(self, on=True):
        """Producer-side push of the versions a rank reads first in a slot (pb2_partition_set_push); call before get()."""
        self._lib.pb2_partition_set_push(self._h, 1 if on else 0)

    def get_push(self, rank, slab_base):
        """(ps_begin[ntasks+1], push[npush]) of `rank` (empty when pushes are off)."""
        n = C.c_int32(0)
        rc = self._lib.pb2_partition_push_count(self._h, rank, C.byref(n))
        if rc != L.PB2_SUCCESS:
            raise L.Pb2Error(rc, "pb2_partition_push_count", "")
        ps_begin = np.zeros(self.sizes(rank)["ntasks"] + 1, np.int32)
        push = np.zeros(n.value, L.PUSH_DTYPE)
        base = np.ascontiguousarray(slab_base, np.uint64)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        rc = self._lib.pb2_partition_get_push(self._h, rank, vp(base), vp(ps_begin), vp(push))
        if rc != L.PB2_SUCCESS:
            raise L.Pb2Error(rc, "pb2_partition_get_push", "")
        return ps_begin, push

    def close(self):
        if self._h:
            self._lib.pb2_partition_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def ex05_global(K_total, NB, world, tile_bytes, kp=1):
    """Ex05_Broadcast (examples/Ex05_Broadcast.jdf:24-58) over `world` ranks as ONE window + owner maps.

    TaskBcast(k) : RW A <- mydata(k), -> A TaskRecv(k, 0..NB..2); runs on rank_of(mydata(k))
    TaskRecv(k,n): READ A <- A TaskBcast(k);                       runs on rank_of(mydata(k + n)) (loc = k + n, :45-47)
    rank_of(mydata(k)) = (k // kp) % world: a 1 x world grid whose k-cyclic factor kp (two_dim_rectangle_cyclic.h: `kp`
    consecutive tiles per rank and cycle; two_dim_rectangle_cyclic.c:281-283) is 1 by default.
    Returns (tasks, succ, tiles, ready, task_rank, tile_rank)."""
    ns = np.arange(0, NB + 1, 2, dtype=np.int32)
    F = len(ns)
    n = K_total * (1 + F)
    t = np.zeros(n, L.TASK_DTYPE)
    t["tile"][:] = -1
    k = np.arange(K_total, dtype=np.int32)
    b = t[:K_total]
    b["body"], b["nb_flows"], b["flags"] = L.BODY_FILL_I32, 1, L.TASK_DEPS_MASK
    b["tile"][:, 0], b["access"][:, 0], b["iparam"][:, 0], b["locals"][:, 0] = k, L.ACCESS_RW, k, k
    b["succ_begin"], b["succ_count"] = k * F, F
    r = t[K_total:]
    kk = np.repeat(k, F)
    r["body"], r["nb_flows"], r["flags"], r["class_id"], r["dep_goal"] = L.BODY_CHECK_I32, 1, L.TASK_DEPS_MASK, 1, 0x1
    r["tile"][:, 0], r["access"][:, 0], r["iparam"][:, 0] = kk, L.ACCESS_READ, kk
    r["locals"][:, 0], r["locals"][:, 1] = kk, np.tile(ns, K_total)
    succ = (K_total + np.arange(K_total * F)).astype(np.uint32)
    tiles = np.zeros(K_total, L.TILE_DTYPE)
    tiles["bytes"], tiles["state"] = tile_bytes, L.TILE_VALID
    owner = lambda x: ((x % K_total) // kp) % world
    task_rank = np.concatenate([owner(k), owner(kk + np.tile(ns, K_total))]).astype(np.int32)
    return t, succ, tiles, np.arange(K_total, dtype=np.int32), task_rank, owner(k).astype(np.int32)


def rtt_global(nt, world, tile_bytes, frags=1):
    """tests/runtime/cuda/rtt.jdf:26-34: PING(k, f), k = 0..NT-1, f = 0..FRAGS-1, RW T <- (k == 0) ? A(f, 0) : T PING(k-1, f),
    placed on A(f, k % WS) with a 1 x WS grid: FRAGS independent chains that hop to the next GPU at every task.
    Every task adds 1 to every element (BASELINE configs[3] body).  Task id = k * frags + f."""
    n = nt * frags
    t = np.zeros(n, L.TASK_DTYPE)
    t["tile"][:] = -1
    i = np.arange(n, dtype=np.int32)
    k, f = i // frags, i % frags
    t["body"], t["nb_flows"], t["flags"] = L.BODY_INCR_I32, 1, L.TASK_DEPS_MASK
    t["iparam"][:, 0] = 1
    t["tile"][:, 0], t["access"][:, 0], t["locals"][:, 0], t["locals"][:, 1] = f, L.ACCESS_RW, k, f
    t["dep_goal"] = np.where(k > 0, 1, 0)
    last = k == nt - 1
    t["succ_count"] = np.where(last, 0, 1)
    t["succ_begin"] = np.minimum(i, n - frags)
    succ = (i[~last] + frags).astype(np.uint32)
    tiles = np.zeros(frags, L.TILE_DTYPE)
    tiles["bytes"], tiles["state"] = tile_bytes, L.TILE_VALID
    return t, succ, tiles, np.arange(frags, dtype=np.int32), (k % world).astype(np.int32), np.zeros(frags, np.int32)


def work_stream(torch):
    """Make a non-default CUDA stream torch's current stream and return its handle: the engine and the NCCL barrier
    are enqueued on it, so "reset -> barrier -> workers" is stream-ordered (the legacy default stream has handle 0,
    which pb2_engine_set_stream reads as "use the engine's own stream")."""
    if torch.cuda.current_stream().cuda_stream == 0:
        torch.cuda.set_stream(torch.cuda.Stream())
    return torch.cuda.current_stream().cuda_stream


def cholesky_global(NT, nb, P, Q, elem_bytes=2):
    """Right-looking tile Cholesky DAG shape (BASELINE configs[4]; the classes of pb2_ptg_cholesky_shape_new):
      POTRF(k)      RW T(k,k)                                  <- SYRK(k,k-1)           body NOP (panel step not modelled)
      TRSM(m,k)     READ T(k,k) x2, RW C(m,k)   m > k          <- POTRF(k), GEMM(m,k,k-1)
      SYRK(m,k)     READ A(m,k) x2, RW T(m,m)   m > k          <- TRSM(m,k), SYRK(m,k-1)
      GEMM(m,n,k)   READ A(m,k), B(n,k), RW C(m,n)  m > n > k  <- TRSM(m,k), TRSM(n,k), GEMM(m,n,k-1)
    GEMM-class bodies C += A * B^T on nb x nb bf16 tiles; owner of a task = rank_of(its RW tile) on a P x Q grid
    (two_dim_rectangle_cyclic.c:281-283).  Tile id of (m,n), m >= n: m*(m+1)/2 + n.  Priorities as bound there:
    POTRF 4(NT-k) > TRSM 3(NT-k) > SYRK 2(NT-k) > GEMM NT-k (used by queue_policy 1 only).
    Returns (tasks, succ, tiles, ready, task_rank, tile_rank)."""
    tid = lambda m, n: m * (m + 1) // 2 + n
    ntiles = NT * (NT + 1) // 2
    ids, rows = {}, []

    def add(cls, m, n, k, body, flows):
        ids[(cls, m, n, k)] = len(rows)
        rows.append((cls, m, n, k, body, flows))

    R, RW = L.ACCESS_READ, L.ACCESS_RW
    for k in range(NT):
        add(0, k, 0, 0, L.BODY_NOP, [(tid(k, k), RW)])
    for k in range(NT):
        for m in range(k + 1, NT):
            add(1, m, k, 0, L.BODY_GEMM_BF16, [(tid(k, k), R), (tid(k, k), R), (tid(m, k), RW)])
    for m in range(1, NT):
        for k in range(m):
            add(2, m, k, 0, L.BODY_GEMM_BF16, [(tid(m, k), R), (tid(m, k), R), (tid(m, m), RW)])
    for m in range(2, NT):
        for n in range(1, m):
            for k in range(n):
                add(3, m, n, k, L.BODY_GEMM_BF16, [(tid(m, k), R), (tid(n, k), R), (tid(m, n), RW)])
    n_t = len(rows)
    t = np.zeros(n_t, L.TASK_DTYPE)
    t["tile"][:] = -1
    edges = [[] for _ in range(n_t)]

    def edge(src, dst_key, flow):
        d = ids.get(dst_key)
        if d is not None:
            edges[src].append((d, flow))

    for i, (cls, m, n, k, body, flows) in enumerate(rows):
        t["body"][i], t["nb_flows"][i], t["class_id"][i], t["flags"][i] = body, len(flows), cls, L.TASK_DEPS_MASK
        for f, (tile, acc) in enumerate(flows):
            t["tile"][i, f], t["access"][i, f] = tile, acc
        t["locals"][i, 0], t["locals"][i, 1] = m, n
        t["iparam"][i] = (nb, nb, nb) if body == L.BODY_GEMM_BF16 else (0, 0, 0)
        t["priority"][i] = (4 * (NT - m), 3 * (NT - n), 2 * (NT - n), NT - k)[cls]     # as the PTG classes bind them
        if cls == 0:                                   # POTRF(k=m) -> TRSM(p, k) flows 0, 1
            for p in range(m + 1, NT):
                edge(i, (1, p, m, 0), 0); edge(i, (1, p, m, 0), 1)
        elif cls == 1:                                 # TRSM(m, k=n)
            kk = n
            edge(i, (2, m, kk, 0), 0); edge(i, (2, m, kk, 0), 1)
            for nn in range(kk + 1, m):
                edge(i, (3, m, nn, kk), 0)
            for p in range(m + 1, NT):
                edge(i, (3, p, m, kk), 1)
        elif cls == 2:                                 # SYRK(m, k=n) -> SYRK(m, k+1) | POTRF(m)
            if n < m - 1:
                edge(i, (2, m, n + 1, 0), 2)
            else:
                edge(i, (0, m, 0, 0), 0)
        else:                                          # GEMM(m, n, k) -> GEMM(m, n, k+1) | TRSM(m, n)
            if k < n - 1:
                edge(i, (3, m, n, k + 1), 2)
            else:
                edge(i, (1, m, n, 0), 2)
    succ, begin = [], np.zeros(n_t, np.int32)
    goal = np.zeros(n_t, np.int32)
    for i, es in enumerate(edges):
        begin[i] = len(succ)
        for d, f in es:
            succ.append((f << 27) | d)
            goal[d] |= 1 << f
    t["succ_begin"], t["succ_count"], t["dep_goal"] = begin, [len(e) for e in edges], goal
    tiles = np.zeros(ntiles, L.TILE_DTYPE)
    tiles["bytes"], tiles["state"] = nb * nb * elem_bytes, L.TILE_VALID
    mm = np.array([m for m in range(NT) for n in range(m + 1)])
    nn = np.array([n for m in range(NT) for n in range(m + 1)])
    tile_rank = ((mm % P) * Q + (nn % Q)).astype(np.int32)
    rw_tile = np.array([r[5][-1][0] for r in rows])
    ready = np.nonzero(goal == 0)[0].astype(np.int32)
    return t, np.array(succ, np.uint32), tiles, ready, tile_rank[rw_tile].astype(np.int32), tile_rank


def translate_remote_targets(part, entries_by_rank):
    """The partitioner names a remote successor by its local task id on the owning rank; that rank's window says how
    to release it (pb2_window_task_entries: index of the dependency word + number of ring entries, in the window's
    own encoding).  entries_by_rank[r] is rank r's table."""
    tgt = part["rs_target"].copy()
    for r, table in enumerate(entries_by_rank):
        m = part["rs_rank"] == r
        if m.any():
            tgt[m] = np.asarray(table)[part["rs_target"][m].astype(np.int64)].astype(np.uint32)
    return tgt


class SharedRun:
    """One rank's half of a window that was split over the GPUs of the box ("direct" path).

    `dist` is torch.distributed (any backend for the handle exchange; the per-step barrier is an all_reduce on
    torch's current CUDA stream, i.e. stream-ordered between the window reset and the worker kernel)."""

    def __init__(self, eng, part, rank, world, dist, torch, kind=0, push=None):
        self.eng, self.rank, self.world, self.dist, self.torch = eng, rank, world, dist, torch
        # producer-side pushes (HBM windows only; the GEMM kernels pull operand slices): opt-in with PB2_MGPU_PUSH=1.
        # Measured r02 (Ex05, 4 GPUs, 1 GiB of ingress per rank and step): pull 2.03 ms, push 2.19 ms -- the transfers run
        # at the rate of a peer copy either way, the push only moves the copy onto the producers' critical path.
        if push is None:
            push = (kind == 0) and os.environ.get("PB2_MGPU_PUSH", "0") == "1"
        part.set_push(push)
        z = part.sizes(rank)
        self.slab_bytes = max(int(z["slab_bytes"]), 256)
        self.slab = eng.malloc(self.slab_bytes, ipc=True)
        eng.h2d(self.slab, np.zeros(self.slab_bytes, np.uint8))
        eng.synchronize()
        handles = [None] * world
        dist.all_gather_object(handles, eng.ipc_export(self.slab))
        self.base = [self.slab if r == rank else eng.ipc_open(handles[r]) for r in range(world)]
        self.p = part.get(rank, self.base)
        eng.set_shared_windows(True, self.p["rs_begin"])
        self.w = eng.window(kind, self.p["tasks"], self.p["succ"], self.p["tiles"], self.p["ready"])
        eng.set_shared_windows(False)
        wh = [None] * world
        dist.all_gather_object(wh, (self.w.export(), self.w.task_entries()))
        tgt = translate_remote_targets(self.p, [h[1] for h in wh])
        self.w.set_remote(rank, [h[0] for h in wh], self.p["rs_begin"], self.p["rs_rank"], tgt)
        self.npush = 0
        if push:
            ps_begin, pushes = part.get_push(rank, self.base)
            self.npush = len(pushes)
            self.w.set_push(ps_begin, pushes)
        self._flag = torch.zeros(1, dtype=torch.int32, device="cuda")
        dist.barrier()

    def slot_of(self, tile):
        """(device address, bytes) of this rank's slot for global tile `tile`, or None if the rank never touches it."""
        hit = np.nonzero(self.p["slot_tile"] == tile)[0]
        if not len(hit):
            return None
        return self.slab + int(self.p["slot_offset"][int(hit[0])])

    def load_home_tiles(self, tile_rank, data):
        """data[tile] (numpy, tile bytes): initial contents; every rank fills the slots of the tiles it is home of."""
        for tile in np.nonzero(np.asarray(tile_rank) == self.rank)[0]:
            addr = self.slot_of(int(tile))
            if addr is not None:
                self.eng.h2d(addr, np.ascontiguousarray(data[int(tile)]))
        self.eng.synchronize()
        self.dist.barrier()

    def read_tile(self, tile, nbytes):
        out = np.empty(nbytes, np.uint8)
        self.eng.d2h(out, self.slot_of(tile))
        self.eng.synchronize()
        return out

    def step(self):
        self.w.arm()                                   # reset dependency words, ring and tile states
        self.dist.all_reduce(self._flag)               # every rank's reset is complete before any worker starts
        self.w.start()

    def wait(self):
        return self.w.wait()


def owner_1xN(k, world):
    """rank_of for a 1 x world grid, kp = kq = 1, ip = jq = 0: tile column k lives on rank k % world."""
    return k % world


def ex05_shard(K_local, NB, world, rank, tile_bytes):
    """Split Ex05_Broadcast (examples/Ex05_Broadcast.jdf:24-58) with nodes = K_local * world over `world` ranks.

    TaskBcast(k) runs on owner(mydata(k)); TaskRecv(k, n) on owner(mydata(k + n)) (loc = k + n, :45-47).
    Returns a dict with
      phase_a : window arrays (tasks, succ, ready, tile ids) of TaskBcast(k) + the receivers that are local
      phase_b : window arrays of the receivers whose tile arrives from another rank
      send_to : ranks that need every tile this rank broadcasts (n even => offsets n % world)
      recv_from : ranks whose tiles this rank's phase-b receivers read, in receive-buffer order
    Local tile l of this rank is global group k = l * world + rank.  Receive buffer j holds the K_local tiles of
    rank recv_from[j], in that rank's local order.
    """
    F = NB // 2 + 1
    offsets = sorted({n % world for n in range(0, NB + 1, 2)})          # (k + n) % world - k % world
    remote_off = [o for o in offsets if o != 0]
    send_to = [(rank + o) % world for o in remote_off]
    recv_from = [(rank - o) % world for o in remote_off]
    ns = np.arange(0, NB + 1, 2)
    local_n = ns[(ns % world) == 0]                                     # receivers of my own tiles that stay here
    # ---- phase A: my TaskBcast + local receivers
    nA = K_local * (1 + len(local_n))
    a = np.zeros(nA, dtype=L.TASK_DTYPE)
    a["tile"][:] = -1
    l = np.arange(K_local, dtype=np.int32)
    kglob = l * world + rank
    b = a[:K_local]
    b["body"], b["nb_flows"], b["flags"] = L.BODY_FILL_I32, 1, L.TASK_DEPS_MASK
    b["tile"][:, 0], b["access"][:, 0], b["iparam"][:, 0], b["locals"][:, 0] = l, L.ACCESS_RW, kglob, kglob
    r = a[K_local:]
    ll = np.repeat(l, len(local_n))
    r["body"], r["nb_flows"], r["flags"], r["class_id"], r["dep_goal"] = L.BODY_CHECK_I32, 1, L.TASK_DEPS_MASK, 1, 0x1
    r["tile"][:, 0], r["access"][:, 0] = ll, L.ACCESS_READ
    r["iparam"][:, 0] = ll * world + rank
    r["locals"][:, 0] = ll * world + rank
    r["locals"][:, 1] = np.tile(local_n, K_local)
    a["succ_begin"][:K_local] = np.arange(K_local) * len(local_n)
    a["succ_count"][:K_local] = len(local_n)
    succ_a = (K_local + np.arange(K_local * len(local_n))).astype(np.uint32)
    # ---- phase B: receivers of tiles that arrive from recv_from[j]
    per_src = []
    for j, (src, off) in enumerate(zip(recv_from, remote_off)):
        n_src = ns[(ns % world) == off]                                 # the n's of rank src's tiles that land here
        nb_ = K_local * len(n_src)
        t = np.zeros(nb_, dtype=L.TASK_DTYPE)
        t["tile"][:] = -1
        ls = np.repeat(l, len(n_src))
        t["body"], t["nb_flows"], t["flags"], t["class_id"], t["dep_goal"] = L.BODY_CHECK_I32, 1, L.TASK_DEPS_MASK, 1, 0
        t["tile"][:, 0], t["access"][:, 0] = j * K_local + ls, L.ACCESS_READ
        t["iparam"][:, 0] = ls * world + src
        t["locals"][:, 0] = ls * world + src
        t["locals"][:, 1] = np.tile(n_src, K_local)
        per_src.append(t)
    bt = np.concatenate(per_src) if per_src else np.zeros(0, L.TASK_DTYPE)
    return {
        "phase_a": dict(tasks=a, succ=succ_a, ready=np.arange(K_local, dtype=np.int32), ntiles=K_local),
        "phase_b": dict(tasks=bt, succ=np.zeros(0, np.uint32), ready=np.arange(len(bt), dtype=np.int32), ntiles=K_local * len(recv_from)),
        "send_to": send_to, "recv_from": recv_from, "F": F, "tile_bytes": tile_bytes,
        "tasks_per_rank": nA + len(bt),
    }


def exchange(dist, send_buf, recv_bufs, send_to, recv_from):
    """One batched send/recv of the whole slab per (destination, source) pair: the PUT of every remote edge."""
    if not send_to:
        return
    ops = []
    for dst in send_to:
        ops.append(dist.P2POp(dist.isend, send_buf, dst))
    for buf, src in zip(recv_bufs, recv_from):
        ops.append(dist.P2POp(dist.irecv, buf, src))
    for w in dist.batch_isend_irecv(ops):
        w.wait()


def ex05_multi_gpu_step_factory(ctx, dev, dc, K, NB, tile_bytes, rank, world, local_rank):
    """Device windows + NCCL exchange for one rank; everything is enqueued on torch's current CUDA stream."""
    import torch
    import torch.distributed as dist
    from .engine import Engine

    sh = ex05_shard(K, NB, world, rank, tile_bytes)
    eng = Engine(local_rank)
    eng.use_stream(work_stream(torch))
    slab = torch.zeros(K * tile_bytes // 4, dtype=torch.int32, device="cuda")
    recv = [torch.empty(K * tile_bytes // 4, dtype=torch.int32, device="cuda") for _ in sh["recv_from"]]

    def tiles_for(bufs):
        n = K * len(bufs)
        t = np.zeros(n, L.TILE_DTYPE)
        for j, b in enumerate(bufs):
            t["dev_ptr"][j * K:(j + 1) * K] = b.data_ptr() + np.arange(K, dtype=np.uint64) * np.uint64(tile_bytes)
        t["bytes"], t["state"] = tile_bytes, L.TILE_VALID
        return t

    pa, pb = sh["phase_a"], sh["phase_b"]
    wa = eng.window(0, pa["tasks"], pa["succ"], tiles_for([slab]), pa["ready"])
    wb = eng.window(0, pb["tasks"], pb["succ"], tiles_for(recv), pb["ready"]) if len(pb["tasks"]) else None
    keep = (eng, slab, recv, wa, wb)

    def step():
        wa.launch()
        exchange(dist, slab, recv, sh["send_to"], sh["recv_from"])
        if wb is not None:
            wb.launch()

    def finish():
        torch.cuda.synchronize()
        st = wa.wait()
        assert st["body_errors"] == 0 and st["tasks_retired"] == len(pa["tasks"])
        if wb is not None:
            st = wb.wait()
            assert st["body_errors"] == 0 and st["tasks_retired"] == len(pb["tasks"]), st
        return keep

    return step, finish, (4 if wb is not None else 2)


def ex05_direct_step_factory(K, NB, tile_bytes, rank, world, local_rank, eng=None, host_tiles=None, kp=1):
    """Ex05 over `world` GPUs, one window per GPU, cross-GPU edges released by the device ("direct" path).

    host_tiles: device-visible alias of this rank's K tiles in pinned host memory (pb2_engine_host_register); when
    given, every step stages the rank's tiles in from host memory inside the kernel (the end-to-end variant)."""
    import torch
    import torch.distributed as dist
    from .engine import Engine

    g = list(ex05_global(K * world, NB, world, tile_bytes, kp))
    if host_tiles is not None:
        assert kp == 1
        tiles = g[2]
        mine = np.nonzero(g[5] == rank)[0]
        tiles["state"][:] = L.TILE_INVALID
        tiles["src_ptr"][mine] = np.uint64(host_tiles) + (mine // world).astype(np.uint64) * np.uint64(tile_bytes)
    part = Partition(*g, nranks=world)
    if eng is None:
        eng = Engine(local_rank)
        eng.use_stream(work_stream(torch))
    run = SharedRun(eng, part, rank, world, dist, torch)
    ntasks = len(run.p["tasks"])

    def finish():
        torch.cuda.synchronize()
        st = run.wait()
        assert st["body_errors"] == 0 and st["tasks_retired"] == ntasks, st
        return run

    return run.step, finish, 3, ntasks
