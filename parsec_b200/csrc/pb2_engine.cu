// pb2_engine.cu -- the persistent sm_90a DAG-execution kernel and its C ABI (include/pb2_engine.h).
//
// What it replaces in the reference (file:line in /root/reference):
//   * the manager thread's check_in_deps / exec / get_data_out / complete_task loop,
//     parsec/mca/device/device_gpu.c:3438-3562, and the 3-stage stream ring of
//     parsec_device_progress_stream (:2592-2731): here every CTA is a worker that pops a task id
//     from a device-resident ring, stages in, runs the body and retires the task itself;
//   * parsec_device_data_stage_in / parsec_default_gpu_stage_in (:1799, :1623): the worker that first
//     touches an INVALID tile moves it (host-pinned or peer memory -> its HBM slot) inside the kernel;
//   * parsec_release_dep_fct -> parsec_release_local_OUT_dependencies -> update_deps_with_counter /
//     _with_mask (parsec/parsec.c:1836, :1749, :1609, :1656): warp 0 of the worker walks the task's
//     out-edges, one lane per edge, atomically decrements / ORs the successor's dependency word and
//     pushes newly-ready successors into the ring with one warp-aggregated tail reservation;
//   * parsec_device_kernel_pop / _epilog (:2943, :3179): pushout flows are copied back to their
//     home location by the worker, versions are bumped for WRITE flows, the task id is appended to the
//     retire log that the host drains in batches to run __parsec_complete_execution bookkeeping.
#include <cuda_runtime.h>
#include <cuda.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include <mutex>
#include <map>
#include <algorithm>
#include <type_traits>

#include "../../include/pb2_engine.h"
#include "pb2_sched.cuh"
#include "pb2_hbm.cuh"
#include "pb2_gemm.cuh"

namespace pb2 {

// ---------------------------------------------------------------------------------------------
// reset: (re)arm one window.  dep words, ring, counters, tile table; the units of a GEMM window.
// ---------------------------------------------------------------------------------------------
// The per-run state of g.w (rearm_run), in a GEMM window its units' words, in a traced window its part records (a zero
// t_pop marks a part that was not popped).  A GEMM window never has more units than tasks.
__global__ void pb2_window_reset_kernel(Win2Dev g, const pb2_tile_t* tiles_init,
                                        const int32_t* ready, int32_t nready) {
    const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t gsz = (size_t)gridDim.x * blockDim.x;
    for (size_t i = gid; i < (size_t)g.nunits; i += gsz) { g.udep[i] = g.units[i].dep_goal; g.parts_left[i] = g.units[i].nparts; }
    if (g.trace.parts)
        for (size_t i = gid; i < (size_t)g.trace.nparts * 8; i += gsz) reinterpret_cast<unsigned long long*>(g.trace.parts)[i] = 0;
    rearm_run(g.w, tiles_init, ready, nready, gid, gsz);
}

// The same bodies as a stand-alone kernel on a caller's stream: what a BODY [type=CUDA] enqueues when it runs under a
// device module that is not ours (the reference's stream engine), see pb2_body_launch.
struct LaunchArgs { void* ptr[PB2_MAX_FLOWS]; unsigned long long bytes[PB2_MAX_FLOWS]; int32_t iparam[3]; float fparam; int32_t body; int32_t nb; };
__device__ unsigned long long g_body_launch_errors;
__global__ void __launch_bounds__(256)
pb2_body_launch_kernel(LaunchArgs la) {
    __shared__ uint32_t red[32];
    __shared__ BodyArgs a;
    // every flow is cut at the same 16-byte aligned offsets, one slice per CTA
    unsigned long long widest = 0;
    for (int f = 0; f < la.nb; ++f) widest = la.bytes[f] > widest ? la.bytes[f] : widest;
    const unsigned long long per = ((widest / gridDim.x) + 15ull) & ~15ull;
    if (threadIdx.x == 0) {
        for (int f = 0; f < PB2_MAX_FLOWS; ++f) {
            const unsigned long long b = f < la.nb ? la.bytes[f] : 0;
            const unsigned long long off = per * blockIdx.x < b ? per * blockIdx.x : b;
            const unsigned long long len = (blockIdx.x == gridDim.x - 1) ? b - off : (off + per <= b ? per : b - off);
            a.flow[f] = f < la.nb ? reinterpret_cast<uint8_t*>(la.ptr[f]) + off : nullptr;
            a.bytes[f] = (uint32_t)len;
            if (f == 0) a.elem0 = (uint32_t)(off >> 2);
        }
        a.part = blockIdx.x; a.iparam[0] = la.iparam[0]; a.iparam[1] = la.iparam[1]; a.iparam[2] = la.iparam[2]; a.fparam = la.fparam;
    }
    __syncthreads();
    const unsigned long long r = run_hbm_body(la.body, a, red);
    if (threadIdx.x == 0 && (la.body == PB2_BODY_CHECK_I32 || la.body == PB2_BODY_CHECK_F32) && (r >> 32))
        atomicAdd(&g_body_launch_errors, r >> 32);
}

struct CopyDesc { void* dst; const void* src; unsigned long long bytes; };

__global__ void __launch_bounds__(256, 4)
pb2_copy_batch_kernel(const CopyDesc* __restrict__ d, int32_t n) {
    for (int32_t i = blockIdx.x; i < n; i += gridDim.x) {
        const CopyDesc c = d[i];
        cta_copy<true>(c.dst, c.src, (size_t)c.bytes);
    }
}

}  // namespace pb2

// =============================================================================================
// Host side
// =============================================================================================
using namespace pb2;

#include "pb2_engine_priv.hpp"
#include "pb2_window_plan.hpp"

// One copy of a window's per-run state: exactly the arrays that rearm_run and pb2_window_reset_kernel write.  alloc_run
// allocates them and run_desc puts them into a launch descriptor; no other host code names them.
struct RunState {
    pb2_tile_t* tiles; int32_t* dep; int32_t* ring; Ctl* ctl; int32_t* retire_log;
    uint32_t* start_seq; uint32_t* end_seq; uint32_t* seen_version; unsigned long long* result; int32_t* worker;
    int32_t* parts_left;                  // RunShape::parts
    uint32_t* slice_claim; uint32_t* slice_done;    // RunShape::claims
    Lanes* lanes;                         // RunShape::lanes
    int32_t* udep; int32_t* unit_parts_left;        // GEMM windows: the units' dependency words and part counts
    pb2_part_trace_t* parts;              // RunShape::trace: part_records of them (TraceDev)
};

struct pb2_window_s {
    pb2_engine_t* e = nullptr;
    int kind = 0;
    int32_t ntasks = 0, ntiles = 0, nready_entries = 0;
    Win2Dev g{};                        // the descriptor without per-run arrays (run_desc adds a copy's)
    RunShape shape;
    pb2_tile_t* d_tiles_init = nullptr;
    int32_t* d_ready = nullptr;         // image of the first nready_entries ring slots
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr;
    bool launched = false;
    bool shared = false;
    WindowKernel kernel;                // what it launches; the linked kernel when a task names a linked body
    // The per-run state by copy.  pb2_window_create fixes ncopies: 2 for a non-shared HBM window with tasks, else 1
    // (DESIGN.md §5).  Copy 0 is allocated at create, copy 1 at the second arm.  Consecutive runs alternate between
    // the copies, and while a run runs, the reset kernel arms the other copy for the next one on the engine's arm
    // stream (ev_arm: its end).  cur: the copy of the last arm; armed: the copy is armed, or will be by work already
    // queued, and no run has used it since; beside: that work is the reset on the arm stream.
    struct Copy { RunState run{}; bool armed = false; bool beside = false; } copy[2];
    int ncopies = 1, cur = 0, arms = 0;
    cudaEvent_t ev_arm = nullptr;
    std::vector<int32_t> task_entry;          // per task: its ring entry with (parts - 1) in the part field
    std::vector<int32_t> task_unit;           // traced windows, per task: the task that leads its scheduling entity
    std::vector<PartEntity> part_entities;   // traced windows: the ring-entry owners by leading task, their records
    std::vector<void*> allocs;
    std::vector<void*> peer_ptrs;
    std::vector<pb2_tile_t*> peer_tiles;     // per rank: its tile table as mapped here (nullptr: none / self)
    std::vector<int32_t> peer_ntiles;
};

// n T (at least one) for window w on `stream`, freed by pb2_window_destroy.
template <class T>
static int dev_alloc(pb2_window_t* w, T** dptr, size_t n, cudaStream_t stream) {
    pb2_engine_t* e = w->e;
    void* p = nullptr;
    // stream-ordered pool allocation: after the first window of a size class this costs microseconds, whereas
    // cudaMalloc/cudaFree next to a slab that fills the device cost hundreds of microseconds each and synchronise the device
    if (w->shared) { PB2_CUDA(e, cudaMalloc(&p, (n ? n : 1) * sizeof(T))); }     // IPC needs cudaMalloc memory
    else PB2_CUDA(e, cudaMallocAsync(&p, (n ? n : 1) * sizeof(T), stream));
    w->allocs.push_back(p);
    *dptr = reinterpret_cast<T*>(p);
    return PB2_SUCCESS;
}

// The same on the upload stream, with host's n T uploaded into them.
template <class T>
static int dev_alloc_copy(pb2_window_t* w, T** dptr, const T* host, size_t n) {
    const int rc = dev_alloc(w, dptr, n, w->e->up_stream);
    if (rc == PB2_SUCCESS && host && n) PB2_CUDA(w->e, cudaMemcpyAsync(*dptr, host, n * sizeof(T), cudaMemcpyHostToDevice, w->e->up_stream));
    return rc;
}

// One tensor map per tile used as a GEMM operand: global tensor [rows][inner] bf16, row pitch inner*2 bytes,
// box {64 (inner, 128 bytes), 128 rows}, 128-byte swizzle: exactly the K-major SWIZZLE_128B smem layout the
// wgmma descriptors in pb2_gemm.cuh describe.  OOB rows/columns of ragged tiles are zero-filled by TMA.
typedef CUresult (*pb2_encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// The tensor maps of a GEMM window, one per tile (zero for a tile that is no operand), from the operand shapes of its plan.
static int encode_tensor_maps(pb2_engine_t* e, const WindowPlan& plan, const pb2_tile_t* tiles, int32_t ntiles,
                              std::vector<CUtensorMap>& maps) {
    static pb2_encode_tiled_fn encode = nullptr;
    if (!encode) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        PB2_CUDA(e, cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
        if (!fn || q != cudaDriverEntryPointSuccess) { e->last_error = "cuTensorMapEncodeTiled not available"; return PB2_ERR_NOT_SUPPORTED; }
        encode = reinterpret_cast<pb2_encode_tiled_fn>(fn);
    }
    maps.resize(ntiles ? ntiles : 1);
    memset(maps.data(), 0, maps.size() * sizeof(CUtensorMap));
    for (int32_t i = 0; i < ntiles; ++i) {
        const int32_t rows = plan.operand_rows[(size_t)i], inner = plan.operand_inner[(size_t)i];
        if (rows == 0) continue;
        cuuint64_t gdim[2] = {(cuuint64_t)inner, (cuuint64_t)rows};
        cuuint64_t gstride[1] = {(cuuint64_t)inner * 2};
        cuuint32_t box[2] = {64, 128};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = encode(&maps[i], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, tiles[i].dev_ptr, gdim, gstride, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { e->last_error = "cuTensorMapEncodeTiled failed"; return PB2_ERR_DEVICE; }
    }
    return PB2_SUCCESS;
}

// The engine's settings a window of `kind` is planned with.
static PlanParams params_of(const pb2_engine_t* e, int kind) {
    PlanParams p;
    p.kind = kind; p.shared = e->shared_windows; p.trace = e->window_trace; p.linked_image = e->linked_module != nullptr;
    p.linked_gemm = e->kernels[1][1][0].fn != nullptr;
    p.queue_policy = e->params.queue_policy; p.gemm_mode = e->params.gemm_mode;
    p.read_groups = e->params.read_groups; p.fuse_readers = e->params.fuse_readers;
    p.nworkers = e->nworkers; p.nworkers_gemm = e->nworkers_gemm;
    p.part_bytes = e->params.part_bytes; p.stage_slice_bytes = e->stage_slice_bytes;
    p.linked_sliceable = e->linked_sliceable; p.linked_checked = e->linked_checked; p.linked_readers = e->linked_readers;
    p.linked_reader_groups = e->linked_reader_groups; p.linked_gemm_bodies = e->linked_gemm_bodies;
    std::copy_n(e->gemm_body_parts, 8, p.gemm_body_parts);
    p.next_rs_begin = e->next_rs_begin;
    return p;
}

// Every array of window w's plan on the device, with the window's initial tile table and, in a GEMM window, its tensor
// maps: allocated and queued on the upload stream, and named in w's descriptor with the scalars the plan fixes.  An
// array the device tests for null is uploaded only when the plan has it.
static int upload_plan(pb2_window_t* w, const WindowPlan& plan, const pb2_tile_t* tiles, const std::vector<CUtensorMap>& tmaps) {
    int rc = PB2_SUCCESS;
    auto up = [&](const auto& v) {
        typename std::decay_t<decltype(v)>::value_type* p = nullptr;
        if (rc == PB2_SUCCESS) rc = dev_alloc_copy(w, &p, v.data(), v.size());
        return p;
    };
    WinDev& d = w->g.w;
    d.tasks = up(plan.tasks);
    d.succ = up(plan.succ);
    if (!plan.group_mem.empty()) { d.group = up(plan.group); d.group_mem = up(plan.group_mem); }
    if (!plan.nparts.empty()) d.nparts = up(plan.nparts);
    if (plan.run.lanes) d.lane = up(plan.lane);
    if (!plan.part_base.empty()) w->g.trace.part_base = up(plan.part_base);
    if (w->kind == 1) {
        w->g.units = up(plan.units); w->g.segs = up(plan.segs); w->g.usucc = up(plan.usucc);
        w->g.tmaps = up(tmaps); w->g.fresh_tmaps = 1;
    }
    w->d_ready = up(plan.ring_image);
    if (rc == PB2_SUCCESS) rc = dev_alloc_copy(w, &w->d_tiles_init, tiles, (size_t)w->ntiles);
    w->nready_entries = (int32_t)plan.ring_image.size();
    w->g.nunits = plan.run.nunits; w->g.trace.nparts = plan.run.part_records;
    d.part_bytes = plan.slice_bytes; d.nlanes = plan.nlanes; d.cap_mask = plan.run.ring - 1;
    return rc;
}

// Copy c of window w's per-run state, sized from w->shape.  pb2_window_create allocates copy 0 on the upload stream,
// and the second pb2_window_arm copy 1, stream-ordered on the engine stream.  The lanes' segment bounds never change:
// both copies hold lane_image's.
static int alloc_run(pb2_window_t* w, int c) {
    pb2_engine_t* e = w->e;
    const RunShape& s = w->shape;
    const cudaStream_t stream = c == 0 ? e->up_stream : e->stream;
    const size_t nt = (size_t)w->ntasks, nl = (size_t)w->ntiles;
    RunState r{};
    int rc = PB2_SUCCESS;
    auto alloc = [&](auto** p, size_t n) { if (rc == PB2_SUCCESS) rc = dev_alloc(w, p, n, stream); };
    alloc(&r.tiles, nl); alloc(&r.dep, nt); alloc(&r.ring, s.ring); alloc(&r.ctl, 1); alloc(&r.retire_log, nt);
    alloc(&r.start_seq, nt); alloc(&r.end_seq, nt); alloc(&r.seen_version, nt * PB2_MAX_FLOWS);
    alloc(&r.result, nt); alloc(&r.worker, nt);
    if (s.parts) alloc(&r.parts_left, nt);
    if (s.claims) { alloc(&r.slice_claim, nl * PB2_SLICE_WORDS); alloc(&r.slice_done, nl * (PB2_SLICE_WORDS + 1)); }
    if (s.lanes) alloc(&r.lanes, 1);
    // every GEMM window has the unit words, even without units: pb2_window_export hands out udep
    if (w->kind == 1) { alloc(&r.udep, (size_t)s.nunits); alloc(&r.unit_parts_left, (size_t)s.nunits); }
    if (s.trace) alloc(&r.parts, (size_t)s.part_records);
    if (rc != PB2_SUCCESS) return rc;
    // copy 1 takes copy 0's lanes device to device: a copy from pageable host memory may wait for the engine stream
    if (s.lanes) PB2_CUDA(e, c == 0 ? cudaMemcpyAsync(r.lanes, &s.lane_image, sizeof(Lanes), cudaMemcpyHostToDevice, stream)
                                    : cudaMemcpyAsync(r.lanes, w->copy[0].run.lanes, sizeof(Lanes), cudaMemcpyDeviceToDevice, stream));
    w->copy[c].run = r;
    return PB2_SUCCESS;
}

// The launch descriptor of copy c of window w: the constant descriptor g with copy c's per-run arrays.
static Win2Dev run_desc(const pb2_window_t* w, int c) {
    const RunState& r = w->copy[c].run;
    Win2Dev g = w->g;
    WinDev& d = g.w;
    d.tiles = r.tiles; d.dep = r.dep; d.ring = r.ring; d.ctl = r.ctl; d.retire_log = r.retire_log;
    d.start_seq = r.start_seq; d.end_seq = r.end_seq; d.seen_version = r.seen_version; d.result = r.result;
    d.worker = r.worker; d.parts_left = r.parts_left; d.slice_claim = r.slice_claim; d.slice_done = r.slice_done;
    d.lanes = r.lanes;
    g.udep = r.udep; g.parts_left = r.unit_parts_left;
    g.trace.parts = r.parts;
    return g;
}

// The part records of the last launch of traced window w, ordered as part_entities (by leading task, then part), with
// task, part and nparts filled in.
static int read_part_records(pb2_window_t* w, std::vector<pb2_part_trace_t>& out) {
    pb2_engine_t* e = w->e;
    std::vector<pb2_part_trace_t> rec((size_t)w->shape.part_records);
    out.clear();
    if (rec.empty()) return PB2_SUCCESS;
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    PB2_CUDA(e, cudaMemcpy(rec.data(), run_desc(w, w->cur).trace.parts, rec.size() * sizeof(pb2_part_trace_t), cudaMemcpyDeviceToHost));
    out.reserve(rec.size());
    for (const PartEntity& pe : w->part_entities)
        for (int32_t p = 0; p < pe.nparts; ++p) {
            out.push_back(rec[(size_t)(pe.base + p)]);
            out.back().task = pe.lead; out.back().part = (uint16_t)p; out.back().nparts = (uint16_t)pe.nparts;
        }
    return PB2_SUCCESS;
}

// ---------------------------------------------------------------------------------------------
// window kernels: the engine's kernel table of the built-in kernels (pb2_window_kernels.cu) and the linked ones, the
// relocatable linked kernels (pb2_engine_linked.cu, pb2_engine_linked_gemm.cu, embedded by pb2_linked_image.S) + the
// application's image, linked by the driver's JIT linker
// ---------------------------------------------------------------------------------------------
extern "C" const unsigned char pb2_linked_engine_image[], pb2_linked_engine_image_end[];
extern "C" const unsigned char pb2_linked_gemm_image[], pb2_linked_gemm_image_end[];
// the same two kernels built with PB2_LINKED_READER_GROUPS, which call pb2_linked_reader_group (PB2_LINK_READER_GROUPS)
extern "C" const unsigned char pb2_linked_engine_groups_image[], pb2_linked_engine_groups_image_end[];
extern "C" const unsigned char pb2_linked_gemm_groups_image[], pb2_linked_gemm_groups_image_end[];
// the GEMM kernel built with PB2_LINKED_GEMM_BODY_ENTRY, without and with PB2_LINKED_READER_GROUPS, which calls
// GEMM-worker bodies through pb2_linked_gemm_body (PB2_LINK_GEMM_BODY_ENTRY)
extern "C" const unsigned char pb2_linked_gemm_entry_image[], pb2_linked_gemm_entry_image_end[];
extern "C" const unsigned char pb2_linked_gemm_entry_groups_image[], pb2_linked_gemm_entry_groups_image_end[];

// The GEMM cubin of a link, by [PB2_LINK_GEMM_BODY_ENTRY][reader groups declared]: its bytes, end and name.
struct LinkedGemmImage { const unsigned char *begin, *end; const char* name; };
static const LinkedGemmImage kLinkedGemmImages[2][2] = {
    {{pb2_linked_gemm_image, pb2_linked_gemm_image_end, "pb2_engine_linked_gemm.cubin"},
     {pb2_linked_gemm_groups_image, pb2_linked_gemm_groups_image_end, "pb2_engine_linked_gemm_groups.cubin"}},
    {{pb2_linked_gemm_entry_image, pb2_linked_gemm_entry_image_end, "pb2_engine_linked_gemm_entry.cubin"},
     {pb2_linked_gemm_entry_groups_image, pb2_linked_gemm_entry_groups_image_end, "pb2_engine_linked_gemm_entry_groups.cubin"}},
};

// The linked window kernels by [kind][(PRIO) + 2 * (TRACE)]: pb2_engine_hbm_kernel<PRIO, TRACE, true>
// (pb2_engine_linked.cu) and pb2_engine_gemm2_kernel<PRIO, TRACE, true> (pb2_engine_linked_gemm.cu)
static const char* const kLinkedKernels[2][4] = {
    {"_ZN3pb221pb2_engine_hbm_kernelILb0ELb0ELb1EEEvNS_6WinDevENS_8TraceDevE",
     "_ZN3pb221pb2_engine_hbm_kernelILb1ELb0ELb1EEEvNS_6WinDevENS_8TraceDevE",
     "_ZN3pb221pb2_engine_hbm_kernelILb0ELb1ELb1EEEvNS_6WinDevENS_8TraceDevE",
     "_ZN3pb221pb2_engine_hbm_kernelILb1ELb1ELb1EEEvNS_6WinDevENS_8TraceDevE"},
    {"_ZN3pb223pb2_engine_gemm2_kernelILb0ELb0ELb1EEEvNS_7Win2DevE",
     "_ZN3pb223pb2_engine_gemm2_kernelILb1ELb0ELb1EEEvNS_7Win2DevE",
     "_ZN3pb223pb2_engine_gemm2_kernelILb0ELb1ELb1EEEvNS_7Win2DevE",
     "_ZN3pb223pb2_engine_gemm2_kernelILb1ELb1ELb1EEEvNS_7Win2DevE"},
};

// The driver calls of the linking point, of every window kernel's launch and of compressible tile memory, fetched
// through the runtime (as cuTensorMapEncodeTiled is): the library gains no link dependency on libcuda.
struct DriverCalls {
    decltype(&cuDeviceGet) device_get = nullptr;
    decltype(&cuDeviceGetAttribute) device_attr = nullptr;
    decltype(&cuMemCreate) mem_create = nullptr;
    decltype(&cuMemGetAllocationGranularity) mem_granularity = nullptr;
    decltype(&cuMemGetAllocationPropertiesFromHandle) mem_props = nullptr;
    decltype(&cuMemAddressReserve) mem_reserve = nullptr;
    decltype(&cuMemMap) mem_map = nullptr;
    decltype(&cuMemSetAccess) mem_set_access = nullptr;
    decltype(&cuMemUnmap) mem_unmap = nullptr;
    decltype(&cuMemAddressFree) mem_address_free = nullptr;
    decltype(&cuMemRelease) mem_release = nullptr;
    bool vmm() const {
        return device_get && device_attr && mem_create && mem_granularity && mem_props && mem_reserve && mem_map &&
               mem_set_access && mem_unmap && mem_address_free && mem_release;
    }
    decltype(&cuLinkCreate) link_create = nullptr;
    decltype(&cuLinkAddData) link_add = nullptr;
    decltype(&cuLinkComplete) link_complete = nullptr;
    decltype(&cuLinkDestroy) link_destroy = nullptr;
    decltype(&cuModuleLoadData) module_load = nullptr;
    decltype(&cuModuleUnload) module_unload = nullptr;
    decltype(&cuModuleGetFunction) get_function = nullptr;
    decltype(&cuFuncGetAttribute) func_attr = nullptr;
    decltype(&cuFuncSetAttribute) func_set_attr = nullptr;
    decltype(&cuOccupancyMaxActiveBlocksPerMultiprocessor) occupancy = nullptr;
    decltype(&cuLaunchKernel) launch = nullptr;
    bool complete() const {
        return link_create && link_add && link_complete && link_destroy && module_load && module_unload && get_function &&
               func_attr && func_set_attr && occupancy && launch;
    }
};

static const DriverCalls& driver() {
    static const DriverCalls d = [] {
        DriverCalls r;
        auto get = [](const char* name, auto& fn) {
            void* p = nullptr;
            cudaDriverEntryPointQueryResult q;
            if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
                fn = reinterpret_cast<std::remove_reference_t<decltype(fn)>>(p);
        };
        get("cuLinkCreate", r.link_create); get("cuLinkAddData", r.link_add); get("cuLinkComplete", r.link_complete);
        get("cuLinkDestroy", r.link_destroy); get("cuModuleLoadData", r.module_load); get("cuModuleUnload", r.module_unload);
        get("cuModuleGetFunction", r.get_function); get("cuFuncGetAttribute", r.func_attr);
        get("cuFuncSetAttribute", r.func_set_attr);
        get("cuOccupancyMaxActiveBlocksPerMultiprocessor", r.occupancy); get("cuLaunchKernel", r.launch);
        get("cuDeviceGet", r.device_get); get("cuDeviceGetAttribute", r.device_attr); get("cuMemCreate", r.mem_create);
        get("cuMemGetAllocationGranularity", r.mem_granularity);
        get("cuMemGetAllocationPropertiesFromHandle", r.mem_props); get("cuMemAddressReserve", r.mem_reserve);
        get("cuMemMap", r.mem_map); get("cuMemSetAccess", r.mem_set_access); get("cuMemUnmap", r.mem_unmap);
        get("cuMemAddressFree", r.mem_address_free); get("cuMemRelease", r.mem_release);
        return r;
    }();
    return d;
}

// Compressible memory on device dev: the L2 compresses its lines on their way to DRAM.
static CUmemAllocationProp compressible_prop(int dev) {
    CUmemAllocationProp p{};
    p.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    p.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    p.location.id = dev;
    p.allocFlags.compressionType = CU_MEM_ALLOCATION_COMP_GENERIC;
    return p;
}

// The granule of compressible memory on device dev, or 0 where the device or the driver offers none.
static size_t compressible_granule(int dev) {
    const DriverCalls& d = driver();
    CUdevice cd = 0;
    int on = 0;
    size_t g = 0;
    if (!d.vmm() || d.device_get(&cd, dev) != CUDA_SUCCESS ||
        d.device_attr(&on, CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED, cd) != CUDA_SUCCESS || !on)
        return 0;
    const CUmemAllocationProp p = compressible_prop(dev);
    return d.mem_granularity(&g, &p, CU_MEM_ALLOC_GRANULARITY_MINIMUM) == CUDA_SUCCESS ? g : 0;
}

static void release_compressible(void* p, CUmemGenericAllocationHandle h, size_t bytes, bool mapped = true) {
    const DriverCalls& d = driver();
    const CUdeviceptr ptr = reinterpret_cast<CUdeviceptr>(p);
    if (mapped) d.mem_unmap(ptr, bytes);
    if (ptr) d.mem_address_free(ptr, bytes);
    d.mem_release(h);
}

// bytes (whole granules) of compressible memory, accessible from the engine's device and from every device that can
// access it as a peer (cudaDeviceEnablePeerAccess does not cover such a mapping), or nullptr with nothing left behind
// when any step fails or the driver grants the memory uncompressed (it does when the compression tags run out).
static void* map_compressible(pb2_engine_t* e, size_t bytes, CUmemGenericAllocationHandle& h) {
    const DriverCalls& d = driver();
    const CUmemAllocationProp p = compressible_prop(e->cuda_device);
    if (d.mem_create(&h, bytes, &p, 0) != CUDA_SUCCESS) return nullptr;
    CUmemAllocationProp got{};
    CUdeviceptr ptr = 0;
    bool mapped = false;
    bool ok = d.mem_props(&got, h) == CUDA_SUCCESS && got.allocFlags.compressionType == CU_MEM_ALLOCATION_COMP_GENERIC;
    if (ok) ok = d.mem_reserve(&ptr, bytes, e->comp_granule, 0, 0) == CUDA_SUCCESS;
    if (ok) ok = mapped = d.mem_map(ptr, bytes, 0, h, 0) == CUDA_SUCCESS;
    if (ok) {
        int ndev = 0;
        if (cudaGetDeviceCount(&ndev) != cudaSuccess) { cudaGetLastError(); ndev = 0; }
        std::vector<CUmemAccessDesc> access;
        for (int dev = 0; dev < ndev; ++dev) {
            int can = dev == e->cuda_device;
            if (!can && cudaDeviceCanAccessPeer(&can, dev, e->cuda_device) != cudaSuccess) { cudaGetLastError(); can = 0; }
            if (can != 1) continue;
            CUmemAccessDesc a{};
            a.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
            a.location.id = dev;
            a.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
            access.push_back(a);
        }
        ok = !access.empty() && d.mem_set_access(ptr, bytes, access.data(), access.size()) == CUDA_SUCCESS;
    }
    if (ok) return reinterpret_cast<void*>(ptr);
    release_compressible(reinterpret_cast<void*>(ptr), h, bytes, mapped);
    return nullptr;
}

// Window kernel fn of `kind` as a kernel table entry k, the same for built-in and linked kernels: its resources, and its
// launch shape.  A GEMM kernel takes the operand ring as dynamic shared memory beside its static shared memory (the
// kernel's, and the bodies' when linked); fits is false when it cannot take the ring or fits no CTA on an SM.  A
// built-in kernel runs on all the engine's workers (nworkers, sized by pb2_engine_create, or nworkers_gemm); a linked
// one on as many of them as fit on the device at once.
static CUresult resolve_kernel(const pb2_engine_t* e, CUfunction fn, int kind, bool linked, WindowKernel& k, bool& fits) {
    const DriverCalls& d = driver();
    const bool gemm = kind == 1;
    const int workers = gemm ? e->nworkers_gemm : e->nworkers;
    k = WindowKernel{};
    k.fn = fn;
    k.block = gemm ? gemm::kThreads : (unsigned)e->params.threads;
    k.dyn_smem = gemm ? gemm::kSmemBytes : 0;
    fits = true;
    CUresult r = d.func_attr(&k.regs, CU_FUNC_ATTRIBUTE_NUM_REGS, fn);
    if (r == CUDA_SUCCESS) r = d.func_attr(&k.local, CU_FUNC_ATTRIBUTE_LOCAL_SIZE_BYTES, fn);
    if (r == CUDA_SUCCESS) r = d.func_attr(&k.static_smem, CU_FUNC_ATTRIBUTE_SHARED_SIZE_BYTES, fn);
    if (r != CUDA_SUCCESS) return r;
    if (gemm && d.func_set_attr(fn, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, gemm::kSmemBytes) != CUDA_SUCCESS) {
        fits = false;
        return CUDA_SUCCESS;
    }
    int occ = 0;
    r = d.occupancy(&occ, fn, (int)k.block, k.dyn_smem);
    if (r == CUDA_SUCCESS && gemm && occ == 0) fits = false;
    k.grid = (unsigned)(linked ? std::max(1, std::min(workers, e->prop.multiProcessorCount * occ)) : workers);
    return r;
}

// The kernel table entry of a window that runs linked bodies or not, of `kind` and variant v: a built-in entry is
// resolved on the current device when a window first needs it.
static int window_kernel(pb2_engine_t* e, bool linked, int kind, int v, WindowKernel& out) {
    static WindowKernelSymbols (*const symbols[4])() = {window_kernels_0, window_kernels_1, window_kernels_2, window_kernels_3};
    std::lock_guard<std::mutex> lk(e->mu);
    WindowKernel& k = e->kernels[linked ? 1 : 0][kind][v];
    if (!k.fn && !linked) {
        if (!driver().complete()) { e->last_error = "the driver's kernel entry points are not available"; return PB2_ERR_NOT_SUPPORTED; }
        const WindowKernelSymbols s = symbols[v]();
        cudaFunction_t fn = nullptr;
        PB2_CUDA(e, cudaGetFuncBySymbol(&fn, kind == 1 ? s.gemm : s.hbm));
        WindowKernel got;
        bool fits = true;
        const CUresult r = resolve_kernel(e, reinterpret_cast<CUfunction>(fn), kind, false, got, fits);
        if (r != CUDA_SUCCESS || !fits) {
            e->last_error = std::string("the built-in ") + (kind == 1 ? "GEMM" : "HBM") + " window kernel cannot run (CUresult " +
                            std::to_string((int)r) + ")";
            return PB2_ERR_DEVICE;
        }
        k = got;
    }
    out = k;
    return PB2_SUCCESS;
}

// What the linker made of the untraced linked kernel of `kind` of the engine's queue policy, and its worker count.
static int linked_info(pb2_engine_t* e, int kind, const char* not_linked, int32_t* regs, int32_t* local_bytes,
                       int32_t* static_smem, int32_t* nworkers) {
    if (!e) return PB2_ERR_BAD_PARAM;
    const WindowKernel& k = e->kernels[1][kind][e->params.queue_policy == 1 ? 1 : 0];
    if (!k.fn) { e->last_error = not_linked; return PB2_ERR_NOT_FOUND; }
    if (regs) *regs = k.regs;
    if (local_bytes) *local_bytes = k.local;
    if (static_smem) *static_smem = k.static_smem;
    if (nworkers) *nworkers = (int32_t)k.grid;
    return PB2_SUCCESS;
}

extern "C" {

int pb2_engine_link_bodies(pb2_engine_t* e, const void* image, size_t bytes, int format, uint32_t sliceable) {
    return pb2_engine_link_bodies_checked(e, image, bytes, format, sliceable, 0);
}

int pb2_engine_link_bodies_checked(pb2_engine_t* e, const void* image, size_t bytes, int format, uint32_t sliceable,
                                   uint32_t checked) {
    return pb2_engine_link_bodies_ex(e, image, bytes, format, sliceable, checked, 0);
}

int pb2_engine_link_bodies_ex(pb2_engine_t* e, const void* image, size_t bytes, int format, uint32_t sliceable,
                              uint32_t checked, uint32_t flags) {
    if (!e) return PB2_ERR_BAD_PARAM;
    if (const char* why = link_args_error(image, bytes, format, sliceable, checked, flags)) { e->last_error = why; return PB2_ERR_BAD_PARAM; }
    const bool gemm_windows = (flags & PB2_LINK_GEMM_WINDOWS) != 0;
    // an image without pb2_linked_reader_group links with the plain kernels, which never name it
    const bool groups = link_reader_groups(flags) != 0;
    const unsigned char* hbm_image = groups ? pb2_linked_engine_groups_image : pb2_linked_engine_image;
    const unsigned char* hbm_end = groups ? pb2_linked_engine_groups_image_end : pb2_linked_engine_image_end;
    // an image without pb2_linked_gemm_body links with GEMM kernels that never name it
    const bool entry = (flags & PB2_LINK_GEMM_BODY_ENTRY) != 0;
    const LinkedGemmImage& gemm_image = kLinkedGemmImages[entry][groups];
    std::lock_guard<std::mutex> lk(e->mu);
    if (e->linked_module) { e->last_error = "the engine has linked an image already (one per engine)"; return PB2_ERR_EXISTS; }
    const DriverCalls& d = driver();
    if (!d.complete()) { e->last_error = "the driver's JIT linker entry points are not available"; return PB2_ERR_NOT_SUPPORTED; }
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    PB2_CUDA(e, cudaFree(nullptr));             // the device's primary context is current: the module is loaded into it
    std::vector<char> err(16384, 0), info(16384, 0);
    CUjit_option opt[] = {CU_JIT_ERROR_LOG_BUFFER, CU_JIT_ERROR_LOG_BUFFER_SIZE_BYTES, CU_JIT_INFO_LOG_BUFFER,
                          CU_JIT_INFO_LOG_BUFFER_SIZE_BYTES, CU_JIT_TARGET};
    void* val[] = {err.data(), reinterpret_cast<void*>((uintptr_t)err.size()), info.data(), reinterpret_cast<void*>((uintptr_t)info.size()),
                   reinterpret_cast<void*>((uintptr_t)CU_TARGET_COMPUTE_90A)};
    std::string ptx;                             // the JIT wants PTX NUL-terminated
    const void* data = image;
    size_t size = bytes;
    if (format == PB2_IMAGE_PTX) { ptx.assign(static_cast<const char*>(image), bytes); data = ptx.c_str(); size = ptx.size() + 1; }
    CUlinkState st = nullptr;
    CUmodule mod = nullptr;
    CUresult r = d.link_create(5, opt, val, &st);
    if (r == CUDA_SUCCESS)
        r = d.link_add(st, CU_JIT_INPUT_CUBIN, const_cast<unsigned char*>(hbm_image), (size_t)(hbm_end - hbm_image),
                       groups ? "pb2_engine_linked_groups.cubin" : "pb2_engine_linked.cubin", 0, nullptr, nullptr);
    if (r == CUDA_SUCCESS && gemm_windows)
        r = d.link_add(st, CU_JIT_INPUT_CUBIN, const_cast<unsigned char*>(gemm_image.begin),
                       (size_t)(gemm_image.end - gemm_image.begin), gemm_image.name, 0, nullptr, nullptr);
    if (r == CUDA_SUCCESS)
        r = d.link_add(st, format == PB2_IMAGE_PTX ? CU_JIT_INPUT_PTX : CU_JIT_INPUT_CUBIN, const_cast<void*>(data), size,
                       "linked bodies", 0, nullptr, nullptr);
    void* out = nullptr;
    size_t out_bytes = 0;
    if (r == CUDA_SUCCESS) r = d.link_complete(st, &out, &out_bytes);
    if (r == CUDA_SUCCESS) r = d.module_load(&mod, out);      // out belongs to the link state: load before destroying it
    if (st) d.link_destroy(st);
    if (r != CUDA_SUCCESS) {
        e->last_error = "linking the application's bodies failed (CUresult " + std::to_string((int)r) + "): " + err.data();
        return PB2_ERR_BAD_PARAM;
    }
    // the linked entries, of GEMM windows only when asked for; a GEMM kernel that does not fit fails the link
    WindowKernel linked[2][4];
    for (int kind = 0; kind < (gemm_windows ? 2 : 1); ++kind)
        for (int v = 0; v < 4; ++v) {
            CUfunction fn = nullptr;
            bool fits = true;
            r = d.get_function(&fn, mod, kLinkedKernels[kind][v]);
            if (r == CUDA_SUCCESS) r = resolve_kernel(e, fn, kind, true, linked[kind][v], fits);
            if (r == CUDA_SUCCESS && fits) continue;
            d.module_unload(mod);
            if (r != CUDA_SUCCESS) {
                e->last_error = std::string("the linked module has no usable ") + (kind == 1 ? "GEMM" : "HBM") +
                                " window kernel (CUresult " + std::to_string((int)r) + ")";
                return PB2_ERR_DEVICE;
            }
            e->last_error = "the linked GEMM window kernel does not fit on an SM: " + std::to_string(linked[kind][v].static_smem) +
                            " bytes of static shared memory (the kernel's and the bodies') beside its " +
                            std::to_string(gemm::kSmemBytes) + " bytes of dynamic shared memory";
            return PB2_ERR_NOT_SUPPORTED;
        }
    e->linked_module = mod;
    std::copy_n(&linked[0][0], 8, &e->kernels[1][0][0]);
    e->linked_sliceable = sliceable; e->linked_checked = checked; e->linked_readers = link_readers(flags);
    e->linked_reader_groups = link_reader_groups(flags); e->linked_gemm_bodies = link_gemm_bodies(flags);
    e->linked_gemm_body_entry = entry;
    return PB2_SUCCESS;
}

int pb2_engine_linked_info(pb2_engine_t* e, int32_t* regs, int32_t* local_bytes, int32_t* static_smem, int32_t* nworkers) {
    return linked_info(e, 0, "the engine has not linked an image (pb2_engine_link_bodies)", regs, local_bytes, static_smem, nworkers);
}

int pb2_engine_linked_gemm_info(pb2_engine_t* e, int32_t* regs, int32_t* local_bytes, int32_t* static_smem, int32_t* nworkers) {
    return linked_info(e, 1, "the engine has not linked the GEMM window kernels (pb2_engine_link_bodies_ex with PB2_LINK_GEMM_WINDOWS)",
                       regs, local_bytes, static_smem, nworkers);
}

int pb2_engine_create(pb2_engine_t** engine, int cuda_device, const pb2_engine_params_t* params) {
    if (!engine) return PB2_ERR_BAD_PARAM;
    *engine = nullptr;
    if (params && params->queue_policy != 0 && params->queue_policy != 1) return PB2_ERR_BAD_PARAM;
    int ndev = 0;
    cudaError_t err = cudaGetDeviceCount(&ndev);
    if (err != cudaSuccess || ndev == 0) {
        // The product path never falls back to a CPU implementation: no GPU => loud failure.
        fprintf(stderr, "pb2_engine_create: no CUDA device (%s)\n", cudaGetErrorString(err));
        return PB2_ERR_DEVICE;
    }
    if (cuda_device < 0 || cuda_device >= ndev) return PB2_ERR_BAD_PARAM;
    pb2_engine_t* e = new pb2_engine_s();
    e->cuda_device = cuda_device;
    PB2_CUDA(e, cudaSetDevice(cuda_device));
    PB2_CUDA(e, cudaGetDeviceProperties(&e->prop, cuda_device));
    if (e->prop.major != 9 || e->prop.minor != 0) {
        fprintf(stderr, "pb2_engine_create: device %d is sm_%d%d; this library only carries sm_90a code\n",
                cuda_device, e->prop.major, e->prop.minor);
        delete e;
        return PB2_ERR_NOT_SUPPORTED;
    }
    pb2_engine_params_t p{};
    if (params) p = *params;
    if (p.workers_per_sm <= 0) p.workers_per_sm = kHbmWorkersPerSm;
    if (p.threads <= 0 || p.threads > PB2_HBM_THREADS) p.threads = PB2_HBM_THREADS;     // the kernel is compiled for this CTA size
    p.threads = (p.threads + 31) & ~31;
    if (p.timeout_ms <= 0) p.timeout_ms = 20000;
    if (p.part_bytes == 0) p.part_bytes = kDefaultPartBytes;
    e->params = p;
    if (const char* sl = getenv("PB2_STAGE_SLICE_BYTES")) e->stage_slice_bytes = atoi(sl);
    if (const char* sm = getenv("PB2_STAGE_MODE")) e->params.stage_mode = atoi(sm);      // 1: SIMT mover (development aid)
    PB2_CUDA(e, cudaStreamCreateWithFlags(&e->own_stream, cudaStreamNonBlocking));
    PB2_CUDA(e, cudaStreamCreateWithFlags(&e->up_stream, cudaStreamNonBlocking));
    PB2_CUDA(e, cudaStreamCreateWithFlags(&e->dma_stream, cudaStreamNonBlocking));
    PB2_CUDA(e, cudaStreamCreateWithFlags(&e->arm_stream, cudaStreamNonBlocking));
    PB2_CUDA(e, cudaEventCreateWithFlags(&e->dma_ev, cudaEventDisableTiming));
    e->stream = e->own_stream;
    e->comp_granule = compressible_granule(cuda_device);
    {   // keep freed window scratch cached in the default mempool instead of returning it to the driver
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, cuda_device) == cudaSuccess) {
            unsigned long long thr = ~0ull;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
        }
    }
    int occ = 0;
    PB2_CUDA(e, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, window_kernels_0().hbm, p.threads, 0));
    int per_sm = occ < p.workers_per_sm ? occ : p.workers_per_sm;
    if (per_sm < 1) per_sm = 1;
    e->nworkers = e->prop.multiProcessorCount * per_sm;
    if (p.max_workers > 0 && p.max_workers < e->nworkers) e->nworkers = p.max_workers;
    e->nworkers_gemm = e->prop.multiProcessorCount;      // one CTA per SM
    if (p.max_workers > 0 && p.max_workers < e->nworkers_gemm) e->nworkers_gemm = p.max_workers;
    *engine = e;
    return PB2_SUCCESS;
}

int pb2_engine_destroy(pb2_engine_t* e) {
    if (!e) return PB2_ERR_BAD_PARAM;
    cudaSetDevice(e->cuda_device);
    for (auto& kv : e->registered) cudaHostUnregister(kv.first);
    if (e->own_stream) cudaStreamDestroy(e->own_stream);
    if (e->up_stream) cudaStreamDestroy(e->up_stream);
    if (e->dma_stream) cudaStreamDestroy(e->dma_stream);
    if (e->arm_stream) cudaStreamDestroy(e->arm_stream);
    if (e->dma_ev) cudaEventDestroy(e->dma_ev);
    if (e->linked_module) driver().module_unload(e->linked_module);
    if (!e->compressible.empty()) cudaDeviceSynchronize();
    for (auto& kv : e->compressible) release_compressible(kv.first, kv.second.first, kv.second.second);
    delete e;
    return PB2_SUCCESS;
}

int pb2_engine_info(pb2_engine_t* e, pb2_engine_info_t* info) {
    if (!e || !info) return PB2_ERR_BAD_PARAM;
    memset(info, 0, sizeof *info);
    info->cuda_device = e->cuda_device;
    info->sm_count = e->prop.multiProcessorCount;
    info->cc_major = e->prop.major; info->cc_minor = e->prop.minor;
    info->nworkers = e->nworkers; info->nworkers_gemm = e->nworkers_gemm;
    info->can_map_host = e->prop.canMapHostMemory;
    size_t f = 0, t = 0;
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    PB2_CUDA(e, cudaMemGetInfo(&f, &t));
    info->total_mem = t; info->free_mem = f;
    info->compression_supported = e->comp_granule != 0;
    info->slab_compressible = e->slab_compressible;
    return PB2_SUCCESS;
}

const char* pb2_engine_last_error(pb2_engine_t* e) { return e ? e->last_error.c_str() : "null engine"; }

int pb2_engine_malloc(pb2_engine_t* e, size_t bytes, void** dev_ptr) { return pb2_engine_malloc_ex(e, bytes, 0, dev_ptr); }

int pb2_engine_malloc_ex(pb2_engine_t* e, size_t bytes, uint32_t flags, void** dev_ptr) {
    if (!e || !dev_ptr || (flags & ~PB2_MALLOC_IPC)) return PB2_ERR_BAD_PARAM;
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    const size_t g = e->comp_granule;
    if (g && bytes >= g) {
        std::lock_guard<std::mutex> lk(e->mu);
        const size_t mapped = (bytes + g - 1) / g * g;
        CUmemGenericAllocationHandle h{};
        void* p = (flags & PB2_MALLOC_IPC) ? nullptr : map_compressible(e, mapped, h);
        e->slab_compressible = p != nullptr;
        if (p) {
            e->compressible[p] = {h, mapped};
            *dev_ptr = p;
            return PB2_SUCCESS;
        }
    }
    cudaError_t err = cudaMalloc(dev_ptr, bytes ? bytes : 16);
    if (err == cudaErrorMemoryAllocation) { cudaGetLastError(); *dev_ptr = nullptr; return PB2_ERR_OUT_OF_RESOURCE; }
    PB2_CUDA(e, err);
    return PB2_SUCCESS;
}

int pb2_engine_free(pb2_engine_t* e, void* dev_ptr) {
    if (!e) return PB2_ERR_BAD_PARAM;
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    std::unique_lock<std::mutex> lk(e->mu);
    auto it = e->compressible.find(dev_ptr);
    if (it == e->compressible.end()) {
        lk.unlock();
        PB2_CUDA(e, cudaFree(dev_ptr));
        return PB2_SUCCESS;
    }
    const auto [h, bytes] = it->second;
    e->compressible.erase(it);
    lk.unlock();
    PB2_CUDA(e, cudaDeviceSynchronize());       // as cudaFree does: work still using the memory ends first
    release_compressible(dev_ptr, h, bytes);
    return PB2_SUCCESS;
}

int pb2_engine_host_register(pb2_engine_t* e, void* host_ptr, size_t bytes, void** dev_alias) {
    if (!e || !host_ptr || !bytes) return PB2_ERR_BAD_PARAM;
    std::lock_guard<std::mutex> lk(e->mu);
    auto it = e->registered.find(host_ptr);
    if (it != e->registered.end()) {   // idempotent, like dc->memory_registration_status
        if (dev_alias) *dev_alias = it->second.second;
        return PB2_SUCCESS;
    }
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    cudaError_t err = cudaHostRegister(host_ptr, bytes, cudaHostRegisterPortable | cudaHostRegisterMapped);
    if (err == cudaErrorHostMemoryAlreadyRegistered) { cudaGetLastError(); }   // e.g. torch pinned memory
    else PB2_CUDA(e, err);
    void* alias = nullptr;
    PB2_CUDA(e, cudaHostGetDevicePointer(&alias, host_ptr, 0));
    if (err != cudaErrorHostMemoryAlreadyRegistered) e->registered[host_ptr] = {bytes, alias};
    if (dev_alias) *dev_alias = alias;
    return PB2_SUCCESS;
}

int pb2_engine_host_unregister(pb2_engine_t* e, void* host_ptr) {
    if (!e) return PB2_ERR_BAD_PARAM;
    std::lock_guard<std::mutex> lk(e->mu);
    auto it = e->registered.find(host_ptr);
    if (it == e->registered.end()) return PB2_ERR_NOT_FOUND;
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    PB2_CUDA(e, cudaHostUnregister(host_ptr));
    e->registered.erase(it);
    return PB2_SUCCESS;
}

int pb2_engine_memcpy_h2d(pb2_engine_t* e, void* dev, const void* host, size_t bytes) {
    if (!e) return PB2_ERR_BAD_PARAM;
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    PB2_CUDA(e, cudaMemcpyAsync(dev, host, bytes, cudaMemcpyHostToDevice, e->stream));
    return PB2_SUCCESS;
}

int pb2_engine_prefetch_h2d(pb2_engine_t* e, void* dev, size_t dev_pitch, const void* host, size_t host_pitch,
                            size_t width_bytes, size_t rows) {
    if (!e || !dev || !host || !width_bytes || !rows) return PB2_ERR_BAD_PARAM;
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    if (rows == 1 || (dev_pitch == width_bytes && host_pitch == width_bytes))
        PB2_CUDA(e, cudaMemcpyAsync(dev, host, width_bytes * rows, cudaMemcpyHostToDevice, e->dma_stream));
    else
        PB2_CUDA(e, cudaMemcpy2DAsync(dev, dev_pitch, host, host_pitch, width_bytes, rows, cudaMemcpyHostToDevice, e->dma_stream));
    e->dma_pending = true;
    return PB2_SUCCESS;
}

int pb2_engine_memcpy_d2h(pb2_engine_t* e, void* host, const void* dev, size_t bytes) {
    if (!e) return PB2_ERR_BAD_PARAM;
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    PB2_CUDA(e, cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, e->stream));
    PB2_CUDA(e, cudaStreamSynchronize(e->stream));
    return PB2_SUCCESS;
}

int pb2_engine_copy_batch(pb2_engine_t* e, void* const* dst, const void* const* src, const uint64_t* bytes, int32_t n) {
    if (!e || n < 0 || (n && (!dst || !src || !bytes))) return PB2_ERR_BAD_PARAM;
    if (n == 0) return PB2_SUCCESS;
    for (int32_t i = 0; i < n; ++i)     // the copy loops index bytes with 32 bits, as tiles are below 4 GiB
        if (bytes[i] >= (1ull << 32)) { e->last_error = "copy of 4 GiB or more"; return PB2_ERR_VALUE_OUT_OF_BOUNDS; }
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    std::vector<CopyDesc> h((size_t)n);
    for (int32_t i = 0; i < n; ++i) h[i] = CopyDesc{dst[i], src[i], bytes[i]};
    CopyDesc* d = nullptr;
    PB2_CUDA(e, cudaMallocAsync(reinterpret_cast<void**>(&d), sizeof(CopyDesc) * (size_t)n, e->stream));
    PB2_CUDA(e, cudaMemcpyAsync(d, h.data(), sizeof(CopyDesc) * (size_t)n, cudaMemcpyHostToDevice, e->stream));
    PB2_CUDA(e, cudaStreamSynchronize(e->stream));     // h is pageable: make sure the staging copy is done
    const int grid = n < e->nworkers ? n : e->nworkers;
    pb2_copy_batch_kernel<<<grid, 256, 0, e->stream>>>(d, n);
    PB2_CUDA(e, cudaGetLastError());
    PB2_CUDA(e, cudaFreeAsync(d, e->stream));
    return PB2_SUCCESS;
}

int pb2_engine_ipc_export(pb2_engine_t* e, void* dev_ptr, unsigned char handle[64]) {
    if (!e || !dev_ptr || !handle) return PB2_ERR_BAD_PARAM;
    {
        std::lock_guard<std::mutex> lk(e->mu);
        auto it = e->compressible.upper_bound(dev_ptr);     // the allocation that holds dev_ptr is the one before
        if (it != e->compressible.begin() &&
            static_cast<char*>(dev_ptr) < static_cast<char*>(std::prev(it)->first) + std::prev(it)->second.second) {
            e->last_error = "the memory is compressible, which CUDA IPC cannot export: allocate memory for other processes "
                            "with pb2_engine_malloc_ex(..., PB2_MALLOC_IPC, ...)";
            return PB2_ERR_NOT_SUPPORTED;
        }
    }
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    cudaIpcMemHandle_t ih;
    PB2_CUDA(e, cudaIpcGetMemHandle(&ih, dev_ptr));
    memcpy(handle, &ih, 64);
    return PB2_SUCCESS;
}
int pb2_engine_ipc_open(pb2_engine_t* e, const unsigned char handle[64], void** dev_ptr) {
    if (!e || !dev_ptr || !handle) return PB2_ERR_BAD_PARAM;
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    cudaIpcMemHandle_t ih;
    memcpy(&ih, handle, 64);
    PB2_CUDA(e, cudaIpcOpenMemHandle(dev_ptr, ih, cudaIpcMemLazyEnablePeerAccess));
    return PB2_SUCCESS;
}
int pb2_engine_ipc_close(pb2_engine_t* e, void* dev_ptr) {
    if (!e || !dev_ptr) return PB2_ERR_BAD_PARAM;
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    PB2_CUDA(e, cudaIpcCloseMemHandle(dev_ptr));
    return PB2_SUCCESS;
}
int pb2_engine_enable_peer(pb2_engine_t* e, int peer_cuda_device) {
    if (!e) return PB2_ERR_BAD_PARAM;
    if (peer_cuda_device == e->cuda_device) return PB2_SUCCESS;
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    int can = 0;
    PB2_CUDA(e, cudaDeviceCanAccessPeer(&can, e->cuda_device, peer_cuda_device));
    if (!can) return PB2_ERR_NOT_SUPPORTED;
    cudaError_t err = cudaDeviceEnablePeerAccess(peer_cuda_device, 0);
    if (err == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); return PB2_SUCCESS; }
    PB2_CUDA(e, err);
    return PB2_SUCCESS;
}

int pb2_body_launch(void* cuda_stream, int body, int nb_args, void* const* ptrs, const uint64_t* bytes,
                    const int32_t* iparam3, float fparam) {
    if (body < 0 || body >= PB2_BODY_MAX || body == PB2_BODY_GEMM_BF16 || body == PB2_BODY_USER) return PB2_ERR_NOT_SUPPORTED;
    if (nb_args < 0 || nb_args > PB2_MAX_FLOWS || (nb_args && (!ptrs || !bytes))) return PB2_ERR_BAD_PARAM;
    LaunchArgs la;
    memset(&la, 0, sizeof la);
    unsigned long long widest = 0;
    for (int f = 0; f < nb_args; ++f) {
        if (bytes[f] >= (1ull << 32)) return PB2_ERR_VALUE_OUT_OF_BOUNDS;
        // the bodies load and store 16-byte vectors
        if (bytes[f] > 0 && (ptrs[f] == nullptr || ((uintptr_t)ptrs[f] & 15))) return PB2_ERR_BAD_PARAM;
        la.ptr[f] = ptrs[f]; la.bytes[f] = bytes[f];
        widest = bytes[f] > widest ? bytes[f] : widest;
    }
    if (iparam3) { la.iparam[0] = iparam3[0]; la.iparam[1] = iparam3[1]; la.iparam[2] = iparam3[2]; }
    la.fparam = fparam; la.body = body; la.nb = nb_args;
    if (body == PB2_BODY_NOP) return PB2_SUCCESS;
    int grid = (int)((widest + 32767) / 32768);             // 32 KiB per CTA
    if (grid < 1) grid = 1;
    if (grid > 1056) grid = 1056;                        // 8 CTAs per SM of an H100 SXM (132 SMs)
    if (body == PB2_BODY_ADD_AT_I32) grid = 1;
    pb2_body_launch_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(cuda_stream)>>>(la);
    return cudaGetLastError() == cudaSuccess ? PB2_SUCCESS : PB2_ERR_DEVICE;
}

int pb2_body_launch_errors(uint64_t* errors, int reset) {
    unsigned long long v = 0;
    if (cudaMemcpyFromSymbol(&v, g_body_launch_errors, sizeof v) != cudaSuccess) return PB2_ERR_DEVICE;
    if (errors) *errors = v;
    if (reset) { v = 0; if (cudaMemcpyToSymbol(g_body_launch_errors, &v, sizeof v) != cudaSuccess) return PB2_ERR_DEVICE; }
    return PB2_SUCCESS;
}

int pb2_engine_set_stage_slice_bytes(pb2_engine_t* e, int32_t bytes) {
    if (!e) return PB2_ERR_BAD_PARAM;
    e->stage_slice_bytes = bytes;
    return PB2_SUCCESS;
}
int pb2_engine_set_part_bytes(pb2_engine_t* e, int32_t part_bytes) {
    if (!e) return PB2_ERR_BAD_PARAM;
    e->params.part_bytes = part_bytes == 0 ? kDefaultPartBytes : part_bytes;
    return PB2_SUCCESS;
}
int pb2_engine_set_gemm_body_parts(pb2_engine_t* e, int body, int32_t nparts) {
    if (!e) return PB2_ERR_BAD_PARAM;
    int rc;
    if (const char* why = gemm_body_parts_error(e->linked_module != nullptr, e->linked_gemm_bodies, body, nparts, &rc)) {
        e->last_error = why;
        return rc;
    }
    e->gemm_body_parts[body - PB2_BODY_LINKED_0] = nparts;
    return PB2_SUCCESS;
}
int pb2_engine_set_window_trace(pb2_engine_t* e, int on) {
    if (!e) return PB2_ERR_BAD_PARAM;
    e->window_trace = on != 0;
    return PB2_SUCCESS;
}
int pb2_engine_set_shared_windows(pb2_engine_t* e, int on, const int32_t* next_rs_begin) {
    if (!e) return PB2_ERR_BAD_PARAM;
    e->shared_windows = on != 0; e->next_rs_begin = on ? next_rs_begin : nullptr;
    return PB2_SUCCESS;
}

int pb2_window_task_entries(pb2_window_t* w, int32_t* entry) {
    if (!w || !entry) return PB2_ERR_BAD_PARAM;
    if ((int32_t)w->task_entry.size() != w->ntasks) return PB2_ERR_NOT_SUPPORTED;
    memcpy(entry, w->task_entry.data(), w->task_entry.size() * sizeof(int32_t));
    return PB2_SUCCESS;
}

int pb2_engine_set_stream(pb2_engine_t* e, void* cuda_stream) {
    if (!e) return PB2_ERR_BAD_PARAM;
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    PB2_CUDA(e, cudaStreamSynchronize(e->stream));
    e->stream = cuda_stream ? reinterpret_cast<cudaStream_t>(cuda_stream) : e->own_stream;
    return PB2_SUCCESS;
}

void* pb2_engine_get_stream(pb2_engine_t* e) { return e ? reinterpret_cast<void*>(e->stream) : nullptr; }

int pb2_engine_synchronize(pb2_engine_t* e) {
    if (!e) return PB2_ERR_BAD_PARAM;
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    PB2_CUDA(e, cudaStreamSynchronize(e->stream));
    return PB2_SUCCESS;
}

// ---------------------------------------------------------------------------------------------
// windows
// ---------------------------------------------------------------------------------------------
int pb2_window_create(pb2_engine_t* e, pb2_window_t** window, int kind,
                      const pb2_task_t* tasks, int32_t ntasks,
                      const uint32_t* succ, int32_t nsucc,
                      const pb2_tile_t* tiles, int32_t ntiles,
                      const int32_t* ready, int32_t nready) {
    if (!e || !window) return PB2_ERR_BAD_PARAM;
    *window = nullptr;
    if ((ntasks && !tasks) || (nsucc && !succ) || (ntiles && !tiles) || (nready && !ready)) return PB2_ERR_BAD_PARAM;
    WindowPlan plan;
    const char* why = nullptr;
    int rc = plan_window(params_of(e, kind), tasks, ntasks, succ, nsucc, tiles, ntiles, ready, nready, plan, &why);
    if (rc != PB2_SUCCESS) {
        if (why) e->last_error = why;
        return rc;
    }
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    WindowKernel kernel;
    if ((rc = window_kernel(e, plan.linked, kind, (plan.run.lanes ? 1 : 0) + (plan.run.trace ? 2 : 0), kernel)) != PB2_SUCCESS) return rc;
    std::vector<CUtensorMap> tmaps;
    if (kind == 1 && (rc = encode_tensor_maps(e, plan, tiles, ntiles, tmaps)) != PB2_SUCCESS) return rc;
    pb2_window_t* w = new pb2_window_s();
    w->kernel = kernel;
    w->shared = e->shared_windows;
    w->e = e; w->kind = kind; w->ntasks = ntasks; w->ntiles = ntiles;
    w->shape = plan.run;
    // shared windows keep one copy (peers hold IPC pointers to it), GEMM windows too (DESIGN.md §5)
    w->ncopies = kind == 0 && !w->shared && ntasks > 0 ? 2 : 1;
    rc = upload_plan(w, plan, tiles, tmaps);
    if (rc == PB2_SUCCESS) rc = alloc_run(w, 0);
    if (rc != PB2_SUCCESS) { pb2_window_destroy(w); return rc; }
    w->task_entry.swap(plan.task_entry);
    w->task_unit.swap(plan.task_unit);
    w->part_entities.swap(plan.part_entities);
    WinDev& d = w->g.w;
    d.shared = w->shared ? 1 : 0; d.ntasks = ntasks; d.ntiles = ntiles; d.stage_mode = e->params.stage_mode;
    d.timeout_ns = (unsigned long long)e->params.timeout_ms * 1000000ull;
    PB2_CUDA(e, cudaEventCreate(&w->ev0));
    PB2_CUDA(e, cudaEventCreate(&w->ev1));
    PB2_CUDA(e, cudaEventCreate(&w->ev2));
    PB2_CUDA(e, cudaEventCreateWithFlags(&w->ev_arm, cudaEventDisableTiming));
    // every descriptor array is on the device when this returns (the host vectors above are temporaries); the
    // upload stream is not ordered behind the engine stream, so creating the next window does not wait for the
    // window that is running
    PB2_CUDA(e, cudaStreamSynchronize(e->up_stream));
    *window = w;
    return PB2_SUCCESS;
}

int pb2_window_destroy(pb2_window_t* w) {
    if (!w) return PB2_ERR_BAD_PARAM;
    cudaSetDevice(w->e->cuda_device);
    if (w->launched) cudaEventSynchronize(w->ev2);        // this window only: a later one may be running
    if (w->copy[0].beside || w->copy[1].beside) cudaEventSynchronize(w->ev_arm);     // a reset of the next run's copy
    for (void* p : w->peer_ptrs) cudaIpcCloseMemHandle(p);
    for (void* p : w->allocs) { if (w->shared) cudaFree(p); else cudaFreeAsync(p, w->e->stream); }
    if (w->ev0) cudaEventDestroy(w->ev0);
    if (w->ev1) cudaEventDestroy(w->ev1);
    if (w->ev2) cudaEventDestroy(w->ev2);
    if (w->ev_arm) cudaEventDestroy(w->ev_arm);
    delete w;
    return PB2_SUCCESS;
}

// The reset kernel over run-state copy c of window w on `stream`, at most per_sm 256-thread CTAs per SM.
static int reset_copy(pb2_window_t* w, int c, cudaStream_t stream, int per_sm) {
    pb2_engine_t* e = w->e;
    const int threads = 256;
    const size_t n = std::max((size_t)w->ntasks, (size_t)w->shape.ring);     // the ring has at least 1024 slots
    const int blocks = (int)std::min((n + threads - 1) / threads, (size_t)e->prop.multiProcessorCount * per_sm);
    pb2_window_reset_kernel<<<blocks, threads, 0, stream>>>(run_desc(w, c), w->d_tiles_init, w->d_ready, w->nready_entries);
    PB2_CUDA(e, cudaGetLastError());
    return PB2_SUCCESS;
}

int pb2_window_arm(pb2_window_t* w) {
    if (!w) return PB2_ERR_BAD_PARAM;
    pb2_engine_t* e = w->e;
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    const int c = w->ncopies == 2 && w->arms > 0 ? w->cur ^ 1 : 0;
    if (!w->copy[c].run.ctl) {
        const int rc = alloc_run(w, c);
        if (rc != PB2_SUCCESS) return rc;
    }
    if (e->dma_pending) {                       // prefetches queued for this window land before its first worker starts
        PB2_CUDA(e, cudaEventRecord(e->dma_ev, e->dma_stream));
        PB2_CUDA(e, cudaStreamWaitEvent(e->stream, e->dma_ev, 0));
        e->dma_pending = false;
    }
    PB2_CUDA(e, cudaEventRecord(w->ev0, e->stream));
    if (!w->copy[c].armed) {
        const int rc = reset_copy(w, c, e->stream, 8);
        if (rc != PB2_SUCCESS) return rc;
    } else if (w->copy[c].beside) {
        // armed beside the last run; a wait here is part of this arm's time (after ev0)
        PB2_CUDA(e, cudaStreamWaitEvent(e->stream, w->ev_arm, 0));
    }
    PB2_CUDA(e, cudaEventRecord(w->ev1, e->stream));
    w->cur = c; w->copy[c].armed = true; w->copy[c].beside = false; w->arms++;
    return PB2_SUCCESS;
}

int pb2_window_start(pb2_window_t* w) {
    if (!w) return PB2_ERR_BAD_PARAM;
    pb2_engine_t* e = w->e;
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    if (w->ntasks > 0) {
        // an HBM kernel takes (WinDev, TraceDev), the trace empty when the window is untraced; a GEMM kernel takes Win2Dev
        Win2Dev g = run_desc(w, w->cur);
        TraceDev tr = w->shape.trace ? g.trace : TraceDev{};
        void* hbm_args[] = {&g.w, &tr};
        void* gemm_args[] = {&g};
        const WindowKernel& k = w->kernel;
        const CUresult r = driver().launch(k.fn, k.grid, 1, 1, k.block, 1, 1, k.dyn_smem, reinterpret_cast<CUstream>(e->stream),
                                           w->kind == 1 ? gemm_args : hbm_args, nullptr);
        if (r != CUDA_SUCCESS) {
            e->last_error = std::string("cuLaunchKernel of the ") + (w->kind == 1 ? "GEMM" : "HBM") + " window kernel failed (CUresult " +
                            std::to_string((int)r) + ")";
            return PB2_ERR_DEVICE;
        }
        if (w->kind == 1) w->g.fresh_tmaps = 0;
    }
    PB2_CUDA(e, cudaEventRecord(w->ev2, e->stream));
    w->launched = true;
    w->copy[w->cur].armed = false;
    const int o = w->cur ^ 1;
    if (w->ncopies == 2 && w->copy[o].run.ctl && !w->copy[o].armed) {
        // The other copy, for the next run, beside this one: after the run that used it last (ev1 of this arm follows
        // it on the engine stream), on one CTA per SM, which fits next to the run's workers (DESIGN.md §5, §6).
        PB2_CUDA(e, cudaStreamWaitEvent(e->arm_stream, w->ev1, 0));
        const int rc = reset_copy(w, o, e->arm_stream, 1);
        if (rc != PB2_SUCCESS) return rc;
        PB2_CUDA(e, cudaEventRecord(w->ev_arm, e->arm_stream));
        w->copy[o].armed = true; w->copy[o].beside = true;
    }
    return PB2_SUCCESS;
}

int pb2_window_launch(pb2_window_t* w) {
    int rc = pb2_window_arm(w);
    return rc == PB2_SUCCESS ? pb2_window_start(w) : rc;
}

int pb2_window_export(pb2_window_t* w, pb2_window_handle_t* h) {
    if (!w || !h) return PB2_ERR_BAD_PARAM;
    pb2_engine_t* e = w->e;
    if (!w->shared) { e->last_error = "window was not created with shared windows enabled"; return PB2_ERR_NOT_SUPPORTED; }
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    memset(h, 0, sizeof *h);
    const Win2Dev g = run_desc(w, 0);           // a shared window's only copy
    cudaIpcMemHandle_t ih;
    PB2_CUDA(e, cudaIpcGetMemHandle(&ih, w->kind == 1 ? g.udep : g.w.dep));  memcpy(h->dep, &ih, 64);   // GEMM windows: unit words
    PB2_CUDA(e, cudaIpcGetMemHandle(&ih, g.w.ring)); memcpy(h->ring, &ih, 64);
    PB2_CUDA(e, cudaIpcGetMemHandle(&ih, g.w.ctl));  memcpy(h->ctl, &ih, 64);
    if (g.w.tiles && w->ntiles > 0) { PB2_CUDA(e, cudaIpcGetMemHandle(&ih, g.w.tiles)); memcpy(h->tiles, &ih, 64); h->ntiles = w->ntiles; }
    h->cap_mask = g.w.cap_mask; h->ntasks = w->ntasks; h->entry_kind = w->kind == 1 ? 1 : 0;
    return PB2_SUCCESS;
}

int pb2_window_set_push(pb2_window_t* w, const int32_t* ps_begin, const pb2_push_t* push, int32_t npush) {
    if (!w || !ps_begin || npush < 0 || (npush && !push)) return PB2_ERR_BAD_PARAM;
    pb2_engine_t* e = w->e;
    if (w->kind == 1 || !w->g.w.peers) { e->last_error = "pushes need an HBM window whose remote edges are set (pb2_window_set_remote)"; return PB2_ERR_NOT_SUPPORTED; }
    if (ps_begin[w->ntasks] != npush) return PB2_ERR_BAD_PARAM;
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    std::vector<PushDev> pd((size_t)npush);
    for (int32_t i = 0; i < npush; ++i) {
        const pb2_push_t& p = push[i];
        if (p.rank < 0 || (size_t)p.rank >= w->peer_tiles.size() || !w->peer_tiles[(size_t)p.rank]) { e->last_error = "push to a rank whose tile table is not mapped"; return PB2_ERR_BAD_PARAM; }
        if (p.desc < 0 || p.desc >= w->peer_ntiles[(size_t)p.rank] || p.src_tile < 0 || p.src_tile >= w->ntiles) { e->last_error = "push descriptor out of bounds"; return PB2_ERR_VALUE_OUT_OF_BOUNDS; }
        memset(&pd[(size_t)i], 0, sizeof(PushDev));
        pd[(size_t)i].dst = reinterpret_cast<void*>(p.dst);
        pd[(size_t)i].dst_state = &w->peer_tiles[(size_t)p.rank][p.desc].state;
        pd[(size_t)i].bytes = p.bytes; pd[(size_t)i].src_tile = p.src_tile;
    }
    int rc;
    int32_t* d_b = nullptr; PushDev* d_p = nullptr;
    if ((rc = dev_alloc_copy(w, &d_b, ps_begin, (size_t)w->ntasks + 1)) != PB2_SUCCESS) return rc;
    if ((rc = dev_alloc_copy(w, &d_p, pd.data(), pd.size())) != PB2_SUCCESS) return rc;
    PB2_CUDA(e, cudaStreamSynchronize(e->up_stream));
    w->g.w.ps_begin = npush ? d_b : nullptr; w->g.w.ps = d_p;
    return PB2_SUCCESS;
}

int pb2_window_set_remote(pb2_window_t* w, int32_t my_rank, int32_t nranks, const pb2_window_handle_t* peers,
                          const int32_t* rs_begin, const int32_t* rs_rank, const uint32_t* rs_target, int32_t nrs) {
    if (!w || nranks <= 0 || my_rank < 0 || my_rank >= nranks || !peers || !rs_begin || nrs < 0) return PB2_ERR_BAD_PARAM;
    pb2_engine_t* e = w->e;
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    const int32_t my_kind = w->kind == 1 ? 1 : 0;
    for (int32_t r = 0; r < nranks; ++r)
        if (r != my_rank && peers[r].entry_kind != my_kind) { e->last_error = "peers run a different kind of window (fused GEMM units vs tasks)"; return PB2_ERR_NOT_SUPPORTED; }
    for (int32_t i = 0; i < nrs; ++i) {
        if (rs_rank[i] < 0 || rs_rank[i] >= nranks || rs_rank[i] == my_rank) { e->last_error = "remote edge to a bad rank"; return PB2_ERR_BAD_PARAM; }
        const int32_t idx = my_kind ? (int32_t)PB2_SUCC_TASK(rs_target[i]) : (int32_t)(rs_target[i] & 0x3FFFFFu);
        if (idx >= peers[rs_rank[i]].ntasks) { e->last_error = "remote edge target out of bounds"; return PB2_ERR_VALUE_OUT_OF_BOUNDS; }
    }
    if (rs_begin[w->ntasks] != nrs) return PB2_ERR_BAD_PARAM;
    std::vector<PeerWin> pw((size_t)nranks);
    for (int32_t r = 0; r < nranks; ++r) {
        memset(&pw[r], 0, sizeof(PeerWin));
        if (r == my_rank) continue;
        void *pd = nullptr, *pr = nullptr, *pc = nullptr, *pt = nullptr;
        cudaIpcMemHandle_t ih;
        memcpy(&ih, peers[r].dep, 64);  PB2_CUDA(e, cudaIpcOpenMemHandle(&pd, ih, cudaIpcMemLazyEnablePeerAccess));
        memcpy(&ih, peers[r].ring, 64); PB2_CUDA(e, cudaIpcOpenMemHandle(&pr, ih, cudaIpcMemLazyEnablePeerAccess));
        memcpy(&ih, peers[r].ctl, 64);  PB2_CUDA(e, cudaIpcOpenMemHandle(&pc, ih, cudaIpcMemLazyEnablePeerAccess));
        memcpy(&ih, peers[r].tiles, 64);
        {   // a window without tiles exports an all-zero handle
            bool any = false;
            for (int b = 0; b < 64; ++b) any |= peers[r].tiles[b] != 0;
            if (any) { PB2_CUDA(e, cudaIpcOpenMemHandle(&pt, ih, cudaIpcMemLazyEnablePeerAccess)); w->peer_ptrs.push_back(pt); }
        }
        w->peer_ptrs.push_back(pd); w->peer_ptrs.push_back(pr); w->peer_ptrs.push_back(pc);
        pw[r].tiles = reinterpret_cast<pb2_tile_t*>(pt);
        w->peer_tiles.resize((size_t)nranks, nullptr); w->peer_tiles[(size_t)r] = reinterpret_cast<pb2_tile_t*>(pt);
        w->peer_ntiles.resize((size_t)nranks, 0); w->peer_ntiles[(size_t)r] = peers[r].ntiles;
        pw[r].dep = reinterpret_cast<int32_t*>(pd); pw[r].ring = reinterpret_cast<int32_t*>(pr);
        pw[r].ctl = reinterpret_cast<Ctl*>(pc); pw[r].cap_mask = peers[r].cap_mask;
    }
    int rc;
    PeerWin* d_pw = nullptr; int32_t* d_b = nullptr; int32_t* d_r = nullptr; uint32_t* d_t = nullptr;
    if ((rc = dev_alloc_copy(w, &d_pw, pw.data(), pw.size())) != PB2_SUCCESS) return rc;
    if ((rc = dev_alloc_copy(w, &d_b, rs_begin, (size_t)w->ntasks + 1)) != PB2_SUCCESS) return rc;
    if ((rc = dev_alloc_copy(w, &d_r, rs_rank, (size_t)nrs)) != PB2_SUCCESS) return rc;
    if ((rc = dev_alloc_copy(w, &d_t, rs_target, (size_t)nrs)) != PB2_SUCCESS) return rc;
    PB2_CUDA(e, cudaStreamSynchronize(e->up_stream));
    w->g.w.peers = d_pw; w->g.w.rs_begin = d_b; w->g.w.rs_rank = d_r; w->g.w.rs_target = d_t; w->g.w.remote_units = my_kind;
    return PB2_SUCCESS;
}

int pb2_window_wait(pb2_window_t* w, pb2_window_stats_t* stats) {
    if (!w) return PB2_ERR_BAD_PARAM;
    pb2_engine_t* e = w->e;
    if (!w->launched) return PB2_ERR_BAD_PARAM;
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    PB2_CUDA(e, cudaEventSynchronize(w->ev2));
    Ctl c;
    PB2_CUDA(e, cudaMemcpy(&c, run_desc(w, w->cur).w.ctl, sizeof c, cudaMemcpyDeviceToHost));
    if (stats) {
        memset(stats, 0, sizeof *stats);
        stats->tasks_retired = c.retired.v;
        stats->bytes_h2d = c.bytes_h2d.v; stats->bytes_d2d = c.bytes_d2d.v; stats->bytes_d2h = c.bytes_d2h.v;
        stats->stage_ins = c.stage_ins.v; stats->body_errors = c.body_errors.v;
        cudaEventElapsedTime(&stats->reset_ms, w->ev0, w->ev1);
        cudaEventElapsedTime(&stats->kernel_ms, w->ev1, w->ev2);
    }
    const int32_t done = (int32_t)c.done.v;
    if (done == kDoneTimeout) { e->last_error = "window watchdog: no task retired within timeout (malformed DAG?)"; return PB2_ERR_DEVICE; }
    if (done == kDoneBadBody) { e->last_error = "window ran a task with an unknown body id"; return PB2_ERR_BAD_PARAM; }
    if ((int64_t)c.retired.v != (int64_t)w->ntasks) { e->last_error = "window ended before all tasks retired"; return PB2_ERROR; }
    return PB2_SUCCESS;
}

int pb2_window_results(pb2_window_t* w, int32_t* retire_order, uint32_t* start_seq, uint32_t* end_seq,
                       uint32_t* seen_version, uint64_t* result, int32_t* worker, pb2_tile_t* tiles_out) {
    if (!w) return PB2_ERR_BAD_PARAM;
    pb2_engine_t* e = w->e;
    PB2_CUDA(e, cudaSetDevice(e->cuda_device));
    const size_t n = (size_t)w->ntasks;
    const WinDev d = run_desc(w, w->cur).w;   // the copy of the last run
    if (retire_order && n) PB2_CUDA(e, cudaMemcpy(retire_order, d.retire_log, n * 4, cudaMemcpyDeviceToHost));
    if (start_seq && n) PB2_CUDA(e, cudaMemcpy(start_seq, d.start_seq, n * 4, cudaMemcpyDeviceToHost));
    if (end_seq && n) PB2_CUDA(e, cudaMemcpy(end_seq, d.end_seq, n * 4, cudaMemcpyDeviceToHost));
    if (seen_version && n) PB2_CUDA(e, cudaMemcpy(seen_version, d.seen_version, n * 4 * PB2_MAX_FLOWS, cudaMemcpyDeviceToHost));
    if (result && n) PB2_CUDA(e, cudaMemcpy(result, d.result, n * 8, cudaMemcpyDeviceToHost));
    if (worker && n) PB2_CUDA(e, cudaMemcpy(worker, d.worker, n * 4, cudaMemcpyDeviceToHost));
    if (tiles_out && w->ntiles) PB2_CUDA(e, cudaMemcpy(tiles_out, d.tiles, (size_t)w->ntiles * sizeof(pb2_tile_t), cudaMemcpyDeviceToHost));
    return PB2_SUCCESS;
}

int pb2_window_trace(pb2_window_t* w, uint64_t* t_start_ns, uint64_t* t_end_ns, uint32_t* smid, int32_t* unit) {
    if (!w) return PB2_ERR_BAD_PARAM;
    pb2_engine_t* e = w->e;
    if (!w->shape.trace) { e->last_error = "window was created without trace (pb2_engine_set_window_trace)"; return PB2_ERR_NOT_SUPPORTED; }
    const size_t n = (size_t)w->ntasks;
    if (unit && n) memcpy(unit, w->task_unit.data(), n * sizeof(int32_t));
    if (!n || (!t_start_ns && !t_end_ns && !smid)) return PB2_SUCCESS;
    std::vector<pb2_part_trace_t> rec;
    const int rc = read_part_records(w, rec);
    if (rc != PB2_SUCCESS) return rc;
    // per leading task, from its entity's parts: the earliest pop, the latest pushout end, the SM of the retiring part
    struct Span { uint64_t t0 = 0, t1 = 0; uint32_t sm = 0; bool retired = false; };
    std::vector<Span> of(n);
    for (const pb2_part_trace_t& r : rec) {
        Span& sp = of[(size_t)r.task];
        if (r.t_pop_ns && (!sp.t0 || r.t_pop_ns < sp.t0)) sp.t0 = r.t_pop_ns;     // 0: not popped
        sp.t1 = std::max(sp.t1, r.t_out_ns);
        if (r.flags & PB2_PART_RETIRED) { sp.sm = r.smid; sp.retired = true; }
    }
    for (size_t t = 0; t < n; ++t) {
        const Span& sp = of[(size_t)w->task_unit[t]];
        if (t_start_ns) t_start_ns[t] = sp.t0;
        if (t_end_ns) t_end_ns[t] = sp.retired ? sp.t1 : 0;
        if (smid) smid[t] = sp.sm;
    }
    return PB2_SUCCESS;
}

int pb2_window_part_trace(pb2_window_t* w, pb2_part_trace_t* out, int32_t cap, int32_t* n) {
    if (!w || !n || cap < 0) return PB2_ERR_BAD_PARAM;
    pb2_engine_t* e = w->e;
    if (!w->shape.trace) { e->last_error = "window was created without trace (pb2_engine_set_window_trace)"; return PB2_ERR_NOT_SUPPORTED; }
    *n = w->shape.part_records;
    if (!out || cap == 0 || *n == 0) return PB2_SUCCESS;
    std::vector<pb2_part_trace_t> rec;
    const int rc = read_part_records(w, rec);
    if (rc != PB2_SUCCESS) return rc;
    memcpy(out, rec.data(), (size_t)std::min(cap, *n) * sizeof(pb2_part_trace_t));
    return PB2_SUCCESS;
}

}  // extern "C"
