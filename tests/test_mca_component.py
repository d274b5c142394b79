"""The real drop-in boundary: parsec/mca/device/b200 compiled INTO the reference runtime (oracle/build_ref_runtime.sh),
driven by task pools the reference's own parsec-ptgpp generated from .jdf files with BODY [type=CUDA] incarnations
(tests/parsec/*.jdf).  CPU tests: the reference runtime alone (CPU bodies: the oracle), and the component in dry-run mode
(scheduling, ownership hand-over, concurrent callers; no bodies run).  GPU tests: the same binaries on an H100, and the
reference's own cuda component on the same task pools as a cross-check."""
import json
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "oracle", "_ref", "bin")


def run(app, args, env=None, timeout=300):
    exe = os.path.join(BIN, app)
    if not os.path.exists(exe):
        pytest.fail(f"{exe} is missing: run __graft_entry__.build() where /root/reference is mounted "
                    "(oracle/build_ref_runtime.sh + make -C tests/parsec)")
    e = dict(os.environ)
    e.pop("PARSEC_MCA_device_b200_enabled", None)
    e.pop("PARSEC_MCA_device_b200_dry_run", None)
    e.update(env or {})
    p = subprocess.run([exe] + [str(a) for a in args], env=e, cwd="/tmp", capture_output=True, text=True, timeout=timeout)
    lines = [l for l in p.stdout.splitlines() if l.startswith("{")]
    assert lines, f"no JSON line from {app}: rc={p.returncode}\n{p.stdout[-2000:]}\n{p.stderr[-2000:]}"
    return p.returncode, json.loads(lines[-1]), p.stderr


CPU_ENV = {"PARSEC_MCA_device_cuda_enabled": "0"}


def test_reference_runtime_cpu_bodies_known_answer():
    """The reference's scheduler + dependency engine + the CPU incarnations: every TaskRecv(k, n) sees k."""
    rc, d, _ = run("ex05_b200", ["-K", 128, "-t", 1024, "-m", "cpu", "-c", 4, "-w"], CPU_ENV)
    assert rc == 0 and d["errors"] == 0 and d["tasks"] == 128 * 9 and d["executed_on_gpu"] == 0
    rc, d, _ = run("stage_b200", ["-m", "cpu"], CPU_ENV)
    assert rc == 0 and d["check_errors"] == 0 and d["host_errors"] == 0


@pytest.mark.parametrize("ndev,cores", [(1, 8), (2, 8), (4, 3)])
def test_component_dry_run_schedules_generated_taskpool(ndev, cores):
    """kernel_scheduler takes every parsec_gpu_task_t the generated hooks build, from concurrent worker threads, and
    completes each task exactly once (the taskpool terminates, executed_tasks adds up)."""
    K, rep = 1024, 3
    rc, d, err = run("ex05_b200", ["-K", K, "-t", 64, "-m", "gpu", "-c", cores, "-r", rep],
                     {"PARSEC_MCA_device_b200_dry_run": str(ndev)})
    assert d["b200_modules"] == ndev and d["gpu_modules"] == ndev, err[-500:]
    assert d["executed_on_gpu"] == K * 9 * rep
    assert d["b200"]["tasks_engine"] == K * 9 * rep and d["b200"]["tasks_lane"] == 0
    assert d["b200"]["manager_entries"] >= 1
    if cores >= 8:
        assert d["b200"]["max_concurrent_callers"] >= 2, "no two worker threads were ever inside kernel_scheduler together"
    # dry-run bodies do not run: the host tiles keep their initial value, every sampled element is 'wrong'
    assert d["errors"] > 0


def test_component_dry_run_memory_pressure_evicts_and_writes_back():
    """A heap of 64 blocks for 256 tiles: clean replicas are evicted, dirty ones written back first."""
    rc, d, err = run("ex05_b200", ["-K", 256, "-t", 131072, "-m", "gpu", "-c", 4],
                     {"PARSEC_MCA_device_b200_dry_run": "1", "PARSEC_MCA_device_b200_memory_number_of_blocks": "64"})
    assert d["executed_on_gpu"] == 256 * 9, err[-500:]
    assert d["b200"]["evictions"] >= 256 - 64
    assert d["b200"]["w2r_copies"] > 0


@pytest.mark.parametrize("knobs", [
    {"parallel_completion": 0},                         # the manager completes every task in line (device_gpu.c:3562-3590)
    {"cmd_slots": 1024},                                # the command ring fills: staged tasks wait for retirements
    {"stage_window": 1},                                # every cold task waits for the one before it
    {"cmd_slots": 1024, "stage_window": 4096, "parallel_completion": 0, "memory_number_of_blocks": 64},
])
def test_component_dry_run_mca_knobs(knobs):
    K, rep = 512, 2
    env = {"PARSEC_MCA_device_b200_dry_run": "1"}
    env.update({"PARSEC_MCA_device_b200_" + k: str(v) for k, v in knobs.items()})
    rc, d, err = run("ex05_b200", ["-K", K, "-t", 131072, "-m", "gpu", "-c", 8, "-r", rep], env, timeout=120)
    assert d["executed_on_gpu"] == K * 9 * rep, err[-500:]


def test_component_dry_run_nvtx_ranges(tmp_path):
    """device_b200_nvtx: the host side of the device as NVTX ranges of the domain "parsec_b200".  nsys is not in the image:
    tests/c/nvtx_counter.c is a minimal NVTX injection library (what a profiler is to the application) that counts them."""
    lib = tmp_path / "libnvtx_counter.so"
    subprocess.run(["gcc", "-shared", "-fPIC", "-O2", "-I/usr/local/cuda/include", "-o", str(lib),
                    os.path.join(ROOT, "tests", "c", "nvtx_counter.c"), "-lpthread"], check=True)
    K = 128
    out = tmp_path / "nvtx.json"
    env = {"PARSEC_MCA_device_b200_dry_run": "1", "NVTX_INJECTION64_PATH": str(lib), "PB2_NVTX_COUNT_FILE": str(out)}
    rc, d, err = run("ex05_b200", ["-K", K, "-t", 1024, "-m", "gpu", "-c", 8], env)            # off by default: no NVTX call at all
    assert d["executed_on_gpu"] == K * 9 and not out.exists(), err[-500:]
    rc, d, err = run("ex05_b200", ["-K", K, "-t", 1024, "-m", "gpu", "-c", 8], dict(env, PARSEC_MCA_device_b200_nvtx="1"))
    assert d["executed_on_gpu"] == K * 9, err[-500:]
    j = json.loads(out.read_text())
    ev = j["events"]
    assert j["domain"] == "parsec_b200" and j["unbalanced_pops"] == 0
    assert j["pops"] == sum(e["pushes"] for e in ev.values())
    assert ev["b200 manager elected"]["marks"] >= 1
    assert ev["b200 start pass"]["pushes"] >= 1 and ev["b200 retire pass"]["pushes"] >= 1
    # a task is completed by an epilog batch of up to four (B200_EPILOG_BATCH) on the worker pool, or in line by the manager
    assert 1 <= ev["b200 epilog batch"]["pushes"] <= K * 9


@pytest.mark.parametrize("ndev", [1, 2])
def test_component_dry_run_several_taskpools_at_once(ndev):
    """Three task pools, each on a collection of its own, handed to the context together: the module sees their tasks
    interleaved (proxies carry the task pool of the task they complete; taskpool_register / unregister per pool)."""
    K, P, rep = 128, 3, 2
    rc, d, _ = run("ex05_b200", ["-K", K, "-t", 1024, "-m", "cpu", "-c", 8, "-w", "-P", P, "-r", rep], CPU_ENV)
    assert rc == 0 and d["errors"] == 0 and d["tasks"] == K * 9 * P and d["pools"] == P
    rc, d, err = run("ex05_b200", ["-K", K, "-t", 1024, "-m", "gpu", "-c", 8, "-P", P, "-r", rep],
                     {"PARSEC_MCA_device_b200_dry_run": str(ndev)}, timeout=120)
    assert d["executed_on_gpu"] == K * 9 * P * rep and d["b200_modules"] == ndev, err[-500:]


@pytest.mark.parametrize("sched", ["ap", "gd", "ip", "lfq", "lhq", "ll", "llp", "ltq", "pbq", "rnd", "spq"])
def test_component_dry_run_under_every_scheduler_module(sched):
    """The completion proxies go through the runtime's scheduler like any task (__parsec_schedule of a ring of tasks with
    priority INT32_MAX): every scheduler module of the reference (parsec/mca/sched/*) has to take them."""
    K, rep = 256, 3
    rc, d, err = run("ex05_b200", ["-K", K, "-t", 1024, "-m", "gpu", "-c", 8, "-r", rep],
                     {"PARSEC_MCA_device_b200_dry_run": "1", "PARSEC_MCA_mca_sched": sched}, timeout=120)
    assert d["executed_on_gpu"] == K * 9 * rep and d["b200_modules"] == 1, err[-500:]


@pytest.mark.parametrize("pins", ["iterators_checker", "print_steals", "alperf"])
def test_component_dry_run_under_pins_modules(pins):
    """(f)4: the runtime's PINS events (EXEC_BEGIN/END around the hook, COMPLETE_EXEC_BEGIN/END inside
    __parsec_complete_execution, scheduling.c:185-192, :477-502) fire for tasks the component runs, and for the proxy
    tasks that carry their completion: the reference's PINS modules run over them unchanged.  iterators_checker walks
    iterate_successors / iterate_predecessors of every task it sees at EXEC_BEGIN."""
    rc, d, err = run("ex05_b200", ["-K", 64, "-t", 1024, "-m", "gpu", "-c", 4],
                     {"PARSEC_MCA_device_b200_dry_run": "1", "PARSEC_MCA_mca_pins": pins})
    assert d["executed_on_gpu"] == 64 * 9 and d["b200_modules"] == 1, err[-500:]


@pytest.mark.gpu
@pytest.mark.parametrize("wb", [False, True])
def test_component_gpu_ex05_known_answer(wb):
    K, rep = 512, 2
    args = ["-K", K, "-t", 65536, "-m", "gpu", "-c", 8, "-r", rep] + (["-w"] if wb else [])
    rc, d, err = run("ex05_b200", args, {"PARSEC_MCA_device_b200_enabled": "1"})
    assert rc == 0, err[-1000:]
    assert d["b200_modules"] == 1 and d["gpu_modules"] == 1
    assert d["errors"] == 0 and d["b200"]["check_mismatches"] == 0
    assert d["executed_on_gpu"] == K * 9 * rep and d["b200"]["tasks_engine"] == K * 9 * rep
    assert d["b200"]["kernel_launches"] >= 1
    # each tile is staged in exactly once per pass that finds it invalid: required == moved (device.c:545-590)
    moved = d["b200"]["bytes_h2d_kernel"] + d["b200"]["bytes_h2d_dma"]
    assert moved == d["h2d_bytes"]
    assert d["h2d_bytes"] == K * 262144 * (1 if wb else rep)


@pytest.mark.gpu
def test_component_gpu_memory_pressure():
    """256 tiles of 256 KiB through a 96-block heap: eviction + write-back on the real device, results still right."""
    rc, d, err = run("ex05_b200", ["-K", 256, "-t", 65536, "-m", "gpu", "-c", 8],
                     {"PARSEC_MCA_device_b200_enabled": "1", "PARSEC_MCA_device_b200_memory_number_of_blocks": "96"})
    assert rc == 0 and d["errors"] == 0 and d["b200"]["check_mismatches"] == 0, err[-1000:]
    assert d["b200"]["evictions"] > 0


@pytest.mark.gpu
def test_component_gpu_stage_callbacks_and_opaque_bodies():
    """Golden vector 'stage' (stage_custom.jdf:266-279): default staging == user stage_in/stage_out == opaque stream body."""
    rc, d, err = run("stage_b200", ["-m", "gpu", "-c", 4], {"PARSEC_MCA_device_b200_enabled": "1"})
    assert rc == 0, err[-1000:]
    assert d["check_errors"] == 0 and d["host_errors"] == 0
    assert d["executed_on_gpu"] == 3 * d["tiles"]
    assert d["tasks_lane"] >= d["tiles"]                    # the opaque bodies ran on the stream lane
    assert d["complete_stage_calls"] == d["tiles"]
    assert d["bytes_h2d_dma"] > 0 and d["bytes_d2h_dma"] > 0  # C is pageable, B is strided: copy engine


@pytest.mark.gpu
def test_reference_cuda_component_agrees_on_the_same_taskpools():
    """The same binaries under the reference's own stream engine (device_cuda): same known answers."""
    env = {"PARSEC_MCA_device_cuda_enabled": "1"}
    rc, d, err = run("ex05_b200", ["-K", 256, "-t", 65536, "-m", "gpu", "-c", 8, "-w"], env)
    assert rc == 0 and d["errors"] == 0 and d["b200_modules"] == 0 and d["gpu_modules"] == 1, err[-1000:]
    rc, d, err = run("stage_b200", ["-m", "gpu", "-c", 4], env)
    assert rc == 0 and d["check_errors"] == 0 and d["host_errors"] == 0, err[-1000:]


def test_component_dry_run_prefetch_advice():
    """PARSEC_DEV_DATA_ADVICE_PREFETCH on every tile before the pool: the DAG itself stages nothing in."""
    rc, d, err = run("ex05_b200", ["-K", 64, "-t", 1024, "-m", "gpu", "-c", 4, "-p"], {"PARSEC_MCA_device_b200_dry_run": "1"})
    assert d["h2d_prefetch_bytes"] == 64 * 4096 and d["h2d_bytes"] == 64 * 4096, err[-500:]
    assert d["executed_on_gpu"] == 64 * 9


@pytest.mark.gpu
def test_component_gpu_prefetch_advice_is_asynchronous_and_valid():
    """The prefetch is an engine task (empty body, one READ flow): the persistent kernel pulls the tiles in; the tasks of
    the pool then find them resident (no second transfer) and the known answer still holds."""
    rc, d, err = run("ex05_b200", ["-K", 256, "-t", 65536, "-m", "gpu", "-c", 8, "-p"], {"PARSEC_MCA_device_b200_enabled": "1"})
    assert rc == 0 and d["errors"] == 0 and d["b200"]["check_mismatches"] == 0, err[-1000:]
    assert d["h2d_prefetch_bytes"] == 256 * 262144 and d["h2d_bytes"] == 256 * 262144
    assert d["b200"]["tasks_engine"] == 256 * 9 + 256           # the 256 prefetch tasks ran in the kernel too


@pytest.mark.gpu
def test_component_two_gpus_in_one_process_peer_pulls():
    """The reference's own multi-GPU model: one process, two device modules.  Readers placed on the other GPU pull the
    producer's replica over NVLink (several readers of one tile arrive together: only the first one's pull may describe
    the tile to the device); the known answer holds and nothing detours through the host."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    rc, d, err = run("ex05_b200", ["-K", 1024, "-t", 65536, "-m", "gpu", "-c", 16, "-r", 2], {"PARSEC_MCA_device_b200_enabled": "2"})
    assert rc == 0 and d["errors"] == 0 and d["b200"]["check_mismatches"] == 0, err[-1000:]
    assert d["b200_modules"] == 2 and d["b200"]["peer_pulls"] > 0 and d["b200"]["peer_detours"] == 0
    rc, d, err = run("stage_b200", ["-m", "gpu", "-c", 4], {"PARSEC_MCA_device_b200_enabled": "2"})
    assert rc == 0 and d["check_errors"] == 0 and d["host_errors"] == 0, err[-1000:]


# ------------------------------------------------------------------------------------------------------------------------
# DTD task pools (parsec_dtd_task_class_add_chore(PARSEC_DEV_CUDA) + parsec_dtd_insert_task_with_task_class) through the
# component: golden vectors of tests/dsl/dtd/dtd_test_cuda_task_insert.c (0xFFFFFFFF), dtd_test_new_tile (2*i) and a
# CPU <-> GPU ping-pong (start + hops)
# ------------------------------------------------------------------------------------------------------------------------
def test_dtd_reference_runtime_cpu_chores_known_answers():
    rc, d, err = run("dtd_b200", ["-C", "-M", 8, "-n", 1024, "-N", 6, "-c", 4], CPU_ENV)
    assert rc == 0 and d["total_errors"] == 0 and d["executed_on_gpu"] == 0, err[-800:]


def test_dtd_component_dry_run_takes_every_dtd_gpu_task():
    """DTD builds the parsec_gpu_task_t (insert_function.c:2393-2425); the component completes each exactly once."""
    M, hops = 8, 6
    rc, d, err = run("dtd_b200", ["-M", M, "-n", 1024, "-N", hops, "-c", 4], {"PARSEC_MCA_device_b200_dry_run": "1"})
    assert d["b200_modules"] == 1, err[-800:]
    # memset: odd tiles; memset_and_read: all; new_tile: two tasks per tile; pingpong: every other hop
    assert d["executed_on_gpu"] == M // 2 + M + 2 * M + M * hops // 2 == d["tasks_engine"]


@pytest.mark.gpu
@pytest.mark.parametrize("opaque", [False, True])
def test_dtd_component_gpu_known_answers(opaque):
    M, hops = 16, 8
    rc, d, err = run("dtd_b200", ["-M", M, "-n", 4096, "-N", hops, "-c", 8] + (["-o"] if opaque else []), {"PARSEC_MCA_device_b200_enabled": "1"})
    assert rc == 0 and d["total_errors"] == 0, (d, err[-1000:])
    assert d["b200_modules"] == 1 and d["executed_on_gpu"] == M // 2 + M + 2 * M + M * hops // 2
    assert d["bytes_h2d_dma"] > 0 and d["bytes_d2h_dma"] > 0        # pageable collection: the copy engine moves it
    if opaque:
        assert d["tasks_lane"] >= M // 2 + M                        # the cudaMemsetAsync bodies ran on the stream lane
    else:
        assert d["tasks_lane"] <= 4                                 # only the first task of each class (it teaches the module its body)


@pytest.mark.gpu
def test_dtd_reference_cuda_component_agrees():
    rc, d, err = run("dtd_b200", ["-M", 16, "-n", 4096, "-N", 8, "-c", 8, "-o"], {"PARSEC_MCA_device_cuda_enabled": "1"})
    assert rc == 0 and d["total_errors"] == 0 and d["b200_modules"] == 0 and d["gpu_modules"] == 1, (d, err[-1000:])


# ------------------------------------------------------------------------------------------------------------------------
# parsec_gpu_task_collect_batch (device_gpu.c:2228-2285): a `batch = true` body takes further staged tasks of its class along
# ------------------------------------------------------------------------------------------------------------------------
def test_batch_reference_runtime_cpu_known_answer():
    rc, d, err = run("batch_b200", ["-m", "cpu", "-M", 32], CPU_ENV)
    assert rc == 0 and d["errors"] == 0 and d["executed_on_gpu"] == 0, err[-800:]


@pytest.mark.gpu
def test_batch_component_gpu_collects_staged_tasks():
    M = 96
    rc, d, err = run("batch_b200", ["-M", M, "-c", 8], {"PARSEC_MCA_device_b200_enabled": "1"})
    assert rc == 0 and d["errors"] == 0, (d, err[-1000:])
    assert d["b200_modules"] == 1 and d["executed_on_gpu"] == M and d["tasks_lane"] == M
    assert d["tasks_in_batches"] == M                       # every task ran exactly once, in some batch
    assert d["max_batch"] > 1 and d["submit_calls"] < M     # and batches did form (up to 5 per the body's callback)
    assert d["lane_batched"] == M - d["submit_calls"]


@pytest.mark.gpu
def test_batch_reference_cuda_component_agrees():
    rc, d, err = run("batch_b200", ["-M", 96, "-c", 8], {"PARSEC_MCA_device_cuda_enabled": "1"})
    assert rc == 0 and d["errors"] == 0 and d["b200_modules"] == 0 and d["tasks_in_batches"] == 96, (d, err[-1000:])


# ------------------------------------------------------------------------------------------------------------------------
# observability: device_b200_trace (what PINS / the profiling keys of device_gpu.c:348-381 report, stamped by the device clock)
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_component_gpu_trace_shows_the_dependency_order_on_the_device_clock(tmp_path):
    K = 128
    base = str(tmp_path / "b200trace")
    rc, d, err = run("ex05_b200", ["-K", K, "-t", 65536, "-m", "gpu", "-c", 8],
                     {"PARSEC_MCA_device_b200_enabled": "1", "PARSEC_MCA_device_b200_trace": base})
    assert rc == 0 and d["errors"] == 0, err[-1000:]
    files = [f for f in os.listdir(tmp_path) if f.startswith("b200trace.") and f.endswith(".json")]
    assert len(files) == 1
    ev = json.load(open(tmp_path / files[0]))["traceEvents"]
    assert len(ev) == K * 9
    bcast_end, nrecv = {}, 0
    for e in ev:
        assert e["ph"] == "X" and e["dur"] > 0 and 0 <= e["tid"] < 160
        if e["name"] == "TaskBcast":
            bcast_end[e["args"]["l0"]] = e["ts"] + e["dur"]
            assert e["args"]["stage_in_bytes"] == 262144                  # the broadcast tile came from the host
    assert len(bcast_end) == K
    for e in ev:
        if e["name"] == "TaskRecv":
            nrecv += 1
            assert e["ts"] >= bcast_end[e["args"]["l0"]] and e["args"]["stage_in_bytes"] == 0   # a receiver starts after its broadcast ended
    assert nrecv == K * 8


@pytest.mark.parametrize("attempt", [0, 1, 2])
def test_component_dry_run_two_devices_with_small_heaps_do_not_wait_for_each_other(attempt):
    """4096 tiles through two heaps of 48 blocks: each heap fills with replicas that only tasks queued on the OTHER device
    still reference.  A task that is short of memory where it is, and whose inputs sit on the peer where it needs none, is
    handed back to the runtime with that peer as its device (this configuration hung two runs in three before)."""
    K = 4096
    rc, d, err = run("ex05_b200", ["-K", K, "-t", 65536, "-m", "gpu", "-c", 3],
                     {"PARSEC_MCA_device_b200_dry_run": "2", "PARSEC_MCA_device_b200_memory_number_of_blocks": "48"}, timeout=120)
    assert d["b200_modules"] == 2 and d["executed_on_gpu"] == K * 9, err[-500:]
    assert d["b200"]["evictions"] > 0
