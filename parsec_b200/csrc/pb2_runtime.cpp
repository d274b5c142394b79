// pb2_runtime.cpp -- host side of the engine: device registry and selection, data coherency, device heap + LRUs,
// the GPU device module (kernel_scheduler -> window building -> launch -> retire/epilog), task completion and
// dependency release.  It mirrors the reference's control flow around the device boundary
//   worker:  __parsec_execute (scheduling.c:126-206) -> chore hook -> dev->kernel_scheduler (device_gpu.c:3375)
//   device:  push (reserve_space :1209, stage_in :1799) -> exec -> pop (:2943) -> epilog (:3179)
//   worker:  __parsec_complete_execution (scheduling.c:469-505) -> release_deps (parsec.c:1836)
// but hands whole dependency-closed sets of GPU tasks ("windows") to the persistent kernel, so the per-task and
// per-edge host round trips of the reference only remain at window boundaries and for CPU incarnations.
#include <algorithm>
#include <chrono>
#include <stdio.h>

#include "pb2_internal.hpp"
#include "pb2_engine_priv.hpp"

static double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
static const bool g_timing = getenv("PB2_TIMING") != nullptr;

// =============================================================================================
// zone heap
// =============================================================================================
void pb2_zone::init(void* base_ptr, int max_seg, size_t unit) {
    base = reinterpret_cast<char*>(base_ptr); unit_size = unit; max_segment = max_seg; clock = 1;
    seg.assign((size_t)max_seg, Seg{UNDEF, 0, 0, 0});
    free_by_size.clear();
    if (max_seg > 0) { seg[0] = Seg{EMPTY, max_seg, 1, 0}; add_free(0); }
}
void pb2_zone::add_free(int tid) { seg[tid].stamp = clock++; free_by_size[Key{seg[tid].nb_units, ~seg[tid].stamp}] = tid; }
void pb2_zone::del_free(int tid) { free_by_size.erase(Key{seg[tid].nb_units, ~seg[tid].stamp}); }

void* pb2_zone::malloc(size_t size) {
    const int nb_units = (int)((size + unit_size - 1) / unit_size);
    if (nb_units == 0 || max_segment == 0) return nullptr;
    auto it = free_by_size.lower_bound(Key{nb_units, 0});        // smallest sufficient size, newest first
    if (it == free_by_size.end()) return nullptr;
    const int tid = it->second;
    free_by_size.erase(it);
    Seg& cur = seg[tid];
    cur.status = FULL;
    if (cur.nb_units > nb_units) {                               // split: the head is allocated
        const int next_tid = tid + cur.nb_units;
        if (next_tid < max_segment) seg[next_tid].nb_prev -= nb_units;
        Seg& nw = seg[tid + nb_units];
        nw.status = EMPTY; nw.nb_prev = nb_units; nw.nb_units = cur.nb_units - nb_units;
        cur.nb_units = nb_units;
        add_free(tid + nb_units);
    }
    return base + (size_t)tid * unit_size;
}

int pb2_zone::free(void* ptr) {
    const ptrdiff_t off = reinterpret_cast<char*>(ptr) - base;
    if (off < 0 || (size_t)off % unit_size) return PB2_ERR_BAD_PARAM;
    int tid = (int)((size_t)off / unit_size);
    if (tid >= max_segment || seg[tid].status == UNDEF) return PB2_ERR_NOT_FOUND;
    if (seg[tid].status == EMPTY) return PB2_ERR_EXISTS;         // double free
    seg[tid].status = EMPTY;
    int prev_tid = tid - seg[tid].nb_prev;
    int next_tid = tid + seg[tid].nb_units;
    if (prev_tid >= 0 && prev_tid < max_segment && prev_tid != tid && seg[prev_tid].status == EMPTY) {
        del_free(prev_tid);
        if (next_tid < max_segment) seg[next_tid].nb_prev += seg[prev_tid].nb_units;
        seg[prev_tid].nb_units += seg[tid].nb_units;
        seg[tid].status = UNDEF;
        tid = prev_tid;
    }
    if (next_tid < max_segment && seg[next_tid].status == EMPTY) {
        del_free(next_tid);
        seg[tid].nb_units += seg[next_tid].nb_units;
        seg[next_tid].status = UNDEF;
        next_tid = tid + seg[tid].nb_units;
        if (next_tid < max_segment) seg[next_tid].nb_prev = seg[tid].nb_units;
    }
    add_free(tid);
    return PB2_SUCCESS;
}

size_t pb2_zone::in_use() const {
    size_t r = 0;
    for (int tid = 0; tid < max_segment; tid += seg[tid].nb_units) {
        if (seg[tid].status == FULL) r += unit_size * (size_t)seg[tid].nb_units;
        if (seg[tid].nb_units <= 0) break;
    }
    return r;
}

// =============================================================================================
// LRU lists (gpu_mem_lru = 1, gpu_mem_owned_lru = 2)
// =============================================================================================
void pb2i_lru_remove(pb2_device_module_t* dev, pb2_data_copy_t* c) {
    const int l = c->lru_list;
    if (!l) return;
    if (c->lru_prev) c->lru_prev->lru_next = c->lru_next; else dev->lru_head[l] = c->lru_next;
    if (c->lru_next) c->lru_next->lru_prev = c->lru_prev; else dev->lru_tail[l] = c->lru_prev;
    c->lru_prev = c->lru_next = nullptr; c->lru_list = 0;
    dev->lru_count[l]--;
}
void pb2i_lru_push_back(pb2_device_module_t* dev, int list, pb2_data_copy_t* c) {
    pb2i_lru_remove(dev, c);
    c->lru_prev = dev->lru_tail[list]; c->lru_next = nullptr;
    if (dev->lru_tail[list]) dev->lru_tail[list]->lru_next = c; else dev->lru_head[list] = c;
    dev->lru_tail[list] = c; c->lru_list = list;
    dev->lru_count[list]++;
}

// =============================================================================================
// data + coherency (parsec/data.c)
// =============================================================================================
static pb2_data_copy_t* new_copy(pb2_data_t* d, int device, uint8_t flags) {
    pb2_data_copy_t* c = new pb2_data_copy_t();
    memset(c, 0, sizeof *c);
    c->device_index = (int8_t)device; c->flags = flags; c->original = d; c->window_tile = -1; c->window_owner = nullptr;
    c->coherency_state = PB2_DATA_COHERENCY_INVALID;
    d->device_copies[device] = c; d->nb_copies++;
    return c;
}
pb2_data_copy_t* pb2i_host_copy(pb2_data_t* d) { return d->device_copies[0]; }

extern "C" {

pb2_data_t* pb2_data_create(pb2_data_collection_t* dc, uint64_t key, void* ptr, size_t size) {
    pb2_data_t* d = new pb2_data_t();
    memset(d, 0, sizeof *d);
    d->owner_device = 0; d->preferred_device = -1; d->key = key; d->dc = dc; d->span = size;
    pb2_data_copy_t* c = new_copy(d, 0, PB2_DATA_FLAG_PARSEC_MANAGED);
    c->coherency_state = PB2_DATA_COHERENCY_OWNED;           // data.c:535
    c->device_private = ptr;
    return d;
}

pb2_data_t* pb2_data_new_temporary(pb2_context_t* ctx, size_t size) {
    (void)ctx;
    // arena NEW datum: host copy exists (arena chunk) but holds nothing of value until a task writes it
    void* mem = nullptr;
    if (posix_memalign(&mem, 64, size ? size : 64)) return nullptr;
    memset(mem, 0, size ? size : 64);
    pb2_data_t* d = pb2_data_create(nullptr, 0, mem, size);
    d->device_copies[0]->flags |= PB2_DATA_FLAG_PARSEC_OWNED;   // we own the host memory
    return d;
}

static void data_destroy(pb2_data_t* d) {
    for (int i = 0; i < PB2_MAX_DEVICES; ++i) {
        pb2_data_copy_t* c = d->device_copies[i];
        if (!c) continue;
        if (i == 0 && (c->flags & PB2_DATA_FLAG_PARSEC_OWNED)) free(c->device_private);
        delete c;
    }
    delete d;
}

// The coherency protocol of a datum when device `device` is about to access it (behaviour of parsec/data.c:334-458,
// checked transition by transition against the reference's own build of that file in tests/test_oracle.py).
// Stated as data: what the DESTINATION replica's state says about fetching, then what the access does to the others.
extern "C++" {
namespace {
enum class Fetch : uint8_t { never, always, if_owner_is_newer };
// indexed by PB2_DATA_COHERENCY_* (INVALID 0, OWNED 1, EXCLUSIVE 2, SHARED 4)
constexpr Fetch kFetchRule[5] = { Fetch::always, Fetch::never, Fetch::never, Fetch::never, Fetch::if_owner_is_newer };

template <class F> inline void for_each_other_valid(pb2_data_t* d, int nb, int skip, F f) {
    for (int i = 0; i < nb; ++i) {
        pb2_data_copy_t* c = d->device_copies[i];
        if (i != skip && c && c->coherency_state != PB2_DATA_COHERENCY_INVALID) f(i, c);
    }
}
}  // namespace
}  // extern "C++"

int pb2_data_start_transfer_ownership_to_copy(pb2_context_t* ctx, pb2_data_t* data, uint8_t device, uint8_t access_mode) {
    const int nb = ctx ? (int)ctx->devices.size() : PB2_MAX_DEVICES;
    pb2_data_copy_t* const dst = data->device_copies[device];
    if (!dst) return PB2_ERR_NOT_FOUND - 100;
    const bool reads = (access_mode & PB2_FLOW_ACCESS_READ) != 0, writes = (access_mode & PB2_FLOW_ACCESS_WRITE) != 0;
    int source = data->owner_device;
    bool fetch = false;

    if (source != device) {                      // a device that owns the datum changes nothing but the book-keeping
        // 1. does the destination need bytes, and from whom?
        switch (kFetchRule[dst->coherency_state & 7]) {
        case Fetch::always:
            fetch = true;
            if (source < 0) for_each_other_valid(data, nb, -1, [&](int i, pb2_data_copy_t*) { source = i; });   // last valid replica
            break;
        case Fetch::if_owner_is_newer:
            for_each_other_valid(data, nb, -1, [&](int, pb2_data_copy_t* c) {
                fetch |= (c->coherency_state == PB2_DATA_COHERENCY_OWNED && c->version > dst->version); });
            break;
        case Fetch::never: break;
        }
        // 2. what the access does to the other replicas
        if (reads) {
            const bool owner_turns_reader = dst->coherency_state == PB2_DATA_COHERENCY_OWNED && !writes;
            for_each_other_valid(data, nb, device, [&](int, pb2_data_copy_t* c) {
                if (owner_turns_reader) {        // the dirty replica is read in place: older replicas die, nobody owns
                    if (c->version < dst->version) c->coherency_state = PB2_DATA_COHERENCY_INVALID;
                    data->owner_device = -1;
                }
                if (c->coherency_state == PB2_DATA_COHERENCY_EXCLUSIVE) c->coherency_state = PB2_DATA_COHERENCY_SHARED;
            });
        } else {
            fetch = false;                       // write-only: the old bytes are not needed
        }
        if (writes) for_each_other_valid(data, nb, -1, [](int, pb2_data_copy_t* c) { c->coherency_state = PB2_DATA_COHERENCY_SHARED; });
    }
    if (reads) dst->readers++;
    if (writes) data->owner_device = (int8_t)device;
    if (!fetch) return -1;
    dst->coherency_state = PB2_DATA_COHERENCY_INVALID;   // until pb2_data_end_transfer_ownership_to_copy
    return source;
}

void pb2_data_end_transfer_ownership_to_copy(pb2_data_t* data, uint8_t device, uint8_t access_mode) {
    pb2_data_copy_t* copy = data->device_copies[device];
    if (!copy) return;
    if (PB2_FLOW_ACCESS_READ & access_mode) copy->coherency_state = PB2_DATA_COHERENCY_SHARED;
    if (PB2_FLOW_ACCESS_WRITE & access_mode) copy->coherency_state = PB2_DATA_COHERENCY_OWNED;
}

/* parsec_data_copy_attach (data.c:174-196): a new, INVALID replica of the datum on `device`; NULL if one exists */
pb2_data_copy_t* pb2_data_copy_attach(pb2_data_t* data, int device) {
    if (!data || device < 0 || device >= PB2_MAX_DEVICES || data->device_copies[device]) return nullptr;
    return new_copy(data, device, PB2_DATA_FLAG_PARSEC_MANAGED);
}

pb2_data_copy_t* pb2_data_get_copy(pb2_data_t* data, int device) {
    return (data && device >= 0 && device < PB2_MAX_DEVICES) ? data->device_copies[device] : nullptr;
}
int pb2_data_copy_state(pb2_data_t* data, int device, int32_t* out) {
    pb2_data_copy_t* c = pb2_data_get_copy(data, device);
    out[0] = c != nullptr;
    if (c) { out[1] = c->coherency_state; out[2] = c->data_transfer_status; out[3] = c->readers; out[4] = (int32_t)c->version; out[5] = c->flags; }
    return PB2_SUCCESS;
}
int pb2_data_owner_device(pb2_data_t* data) { return data->owner_device; }
int pb2_data_preferred_device(pb2_data_t* data) { return data->preferred_device; }

// =============================================================================================
// context, MCA parameters, device registry (device.c)
// =============================================================================================
int pb2_init(pb2_context_t** pctx, int nb_cores) {
    if (!pctx) return PB2_ERR_BAD_PARAM;
    pb2_context_t* ctx = new pb2_context_s();
    ctx->nb_cores = nb_cores > 0 ? nb_cores : 1;
    // defaults: device.c:342-363, device_cuda_component.c:135-178
    ctx->mca["device_load_balance_skew"] = 20;
    ctx->mca["device_load_balance_allow_cpu"] = 0;
    ctx->mca["device_show_statistics"] = 0;
    ctx->mca["device_cuda_memory_use"] = 95;
    ctx->mca["device_cuda_memory_block_size"] = 512 * 1024;
    ctx->mca["device_cuda_memory_number_of_blocks"] = -1;
    ctx->mca["device_cuda_max_number_of_ejected_data"] = 20;
    ctx->mca["device_engine_workers_per_sm"] = 0;
    ctx->mca["device_engine_max_workers"] = 0;
    ctx->mca["device_engine_timeout_ms"] = 0;
    ctx->mca["device_engine_gemm_mode"] = 0;
    // 1: windows pop ready tasks by priority (JDF priority expressions, DTD insert priorities), FIFO among equals
    ctx->mca["device_engine_queue_policy"] = 0;
    // 1: windows record when and on which SM each task ran (pb2_taskpool_device_trace), through the traced kernels
    ctx->mca["device_engine_trace"] = 0;
    // a batch of at least _min_roots ready GPU tasks is cut into _pipeline windows of whole dependency closures:
    // while one window runs, the host builds the next one and replays the bookkeeping of the previous one
    // tiles a window has to read from pinned host memory: runs of at least this many contiguous bytes (host and
    // device side) go through the copy engine before the window starts, the rest is staged by the worker CTAs
    ctx->mca["device_engine_dma_prefetch_min_bytes"] = 1 << 20;      // 0 disables
    ctx->mca["device_engine_pipeline"] = 4;
    ctx->mca["device_engine_pipeline_min_roots"] = 2048;
    // index 0: the CPU; index 1: the recursive pseudo-device (device.c:1041-1110)
    for (int i = 0; i < 2; ++i) {
        pb2_device_module_t* d = new pb2_device_module_s();
        d->ctx = ctx; d->device_index = (uint8_t)i; d->type = i == 0 ? PB2_DEV_CPU : PB2_DEV_RECURSIVE;
        d->name = i == 0 ? "cpu" : "recursive";
        d->st.gflops_fp16 = d->st.gflops_fp32 = 100; d->st.gflops_tf32 = 100; d->st.gflops_fp64 = 50;   // per core
        ctx->devices.push_back(d);
    }
    *pctx = ctx;
    return PB2_SUCCESS;
}

int pb2_mca_param_set_int(pb2_context_t* ctx, const char* name, int64_t value) {
    if (!ctx || !name) return PB2_ERR_BAD_PARAM;
    if (!ctx->mca.count(name)) return PB2_ERR_NOT_FOUND;
    ctx->mca[name] = value;
    return PB2_SUCCESS;
}
int pb2_mca_param_get_int(pb2_context_t* ctx, const char* name, int64_t* value) {
    if (!ctx || !name || !value) return PB2_ERR_BAD_PARAM;
    auto it = ctx->mca.find(name);
    if (it == ctx->mca.end()) return PB2_ERR_NOT_FOUND;
    *value = it->second;
    return PB2_SUCCESS;
}

int pb2_device_cuda_module_init(pb2_context_t* ctx, int cuda_index, int dry_run, pb2_device_module_t** module) {
    if (!ctx || !module) return PB2_ERR_BAD_PARAM;
    *module = nullptr;
    if (ctx->devices_frozen) return PB2_ERR_NOT_SUPPORTED;              // device.c:1117
    if (ctx->devices.size() >= PB2_MAX_DEVICES) return PB2_ERR_OUT_OF_RESOURCE;
    pb2_device_module_t* d = new pb2_device_module_s();
    d->ctx = ctx; d->type = PB2_DEV_CUDA; d->cuda_index = cuda_index; d->dry_run = dry_run != 0;
    d->device_index = (uint8_t)ctx->devices.size();
    char nm[64]; snprintf(nm, sizeof nm, "cuda(%d)", cuda_index); d->name = nm;
    d->mem_block_size = (size_t)ctx->mca["device_cuda_memory_block_size"];
    d->trace = ctx->mca["device_engine_trace"] != 0;
    size_t total = 0, freeb = 0;
    if (!d->dry_run) {
        pb2_engine_params_t p{};
        p.workers_per_sm = (int32_t)ctx->mca["device_engine_workers_per_sm"];
        p.max_workers = (int32_t)ctx->mca["device_engine_max_workers"];
        p.timeout_ms = (int32_t)ctx->mca["device_engine_timeout_ms"];
        p.gemm_mode = (int32_t)ctx->mca["device_engine_gemm_mode"];
        p.queue_policy = (int32_t)ctx->mca["device_engine_queue_policy"];
        int rc = pb2_engine_create(&d->engine, cuda_index, &p);
        if (rc != PB2_SUCCESS) { delete d; return rc; }                 // no GPU => loud failure, no fallback
        if (d->trace) pb2_engine_set_window_trace(d->engine, 1);
        pb2_engine_info_t info;
        pb2_engine_info(d->engine, &info);
        d->major = info.cc_major; d->minor = info.cc_minor;
        total = info.total_mem; freeb = info.free_mem;
    } else {
        d->major = 9; d->minor = 0;
        total = freeb = (size_t)1 << 30;
    }
    // dense GFLOP/s of one H100 SXM (data sheet), the sm_90 rates of the reference's table (device_cuda_module.c:45-142)
    d->st.gflops_fp16 = 989000; d->st.gflops_tf32 = 495000; d->st.gflops_fp32 = 67000; d->st.gflops_fp64 = 34000;
    // parsec_device_memory_reserve, device_gpu.c:866-991
    int64_t nblocks = ctx->mca["device_cuda_memory_number_of_blocks"];
    if (nblocks <= 0) nblocks = (int64_t)((double)freeb * (double)ctx->mca["device_cuda_memory_use"] / 100.0 / (double)d->mem_block_size);
    if (nblocks < 1) nblocks = 1;
    if (nblocks > 0x7fffffff) nblocks = 0x7fffffff;
    d->mem_nb_blocks = nblocks;
    if (!d->dry_run) {
        int rc = PB2_ERR_OUT_OF_RESOURCE;
        while (d->mem_nb_blocks > 0) {
            rc = pb2_engine_malloc(d->engine, (size_t)d->mem_nb_blocks * d->mem_block_size, &d->slab);
            if (rc == PB2_SUCCESS) break;
            if (rc != PB2_ERR_OUT_OF_RESOURCE) break;
            d->mem_nb_blocks = d->mem_nb_blocks * 9 / 10;               // back off like the reference's retry loop
        }
        if (rc != PB2_SUCCESS) { pb2_engine_destroy(d->engine); delete d; return rc; }
    } else {
        d->slab = reinterpret_cast<void*>((uintptr_t)0x100000000ull * (uintptr_t)(d->device_index));
    }
    d->zone.init(d->slab, (int)d->mem_nb_blocks, d->mem_block_size);
    ctx->devices.push_back(d);
    *module = d;
    (void)total;
    return PB2_SUCCESS;
}

int pb2_mca_device_registration_complete(pb2_context_t* ctx) {
    if (!ctx) return PB2_ERR_BAD_PARAM;
    if (ctx->devices_frozen) return PB2_ERR_NOT_SUPPORTED;
    ctx->devices_frozen = true;
    int64_t total64 = 0;
    for (auto* d : ctx->devices) {
        if (d->type & PB2_DEV_RECURSIVE) continue;
        // all_devices_attached: peer access matrix (device_cuda_module.c:144-181).  One process drives all the
        // GPUs here, NVSwitch connects every pair: all GPU pairs are peers.
        if (PB2_DEV_IS_GPU(d->type))
            for (auto* o : ctx->devices) if (PB2_DEV_IS_GPU(o->type)) d->peer_access_mask |= 1u << o->device_index;
        const int64_t c = (d->type & PB2_DEV_CPU) ? ctx->nb_cores : 1;
        total64 += c * d->st.gflops_fp64;
    }
    for (auto* d : ctx->devices) {
        if (d->type & PB2_DEV_RECURSIVE) continue;
        d->st.time_estimate_default = (int64_t)((double)total64 / (double)d->st.gflops_fp64);   // device.c:827
    }
    return PB2_SUCCESS;
}

int pb2_nb_devices(pb2_context_t* ctx) { return ctx ? (int)ctx->devices.size() : 0; }
pb2_device_module_t* pb2_mca_device_get(pb2_context_t* ctx, int idx) {
    return (ctx && idx >= 0 && idx < (int)ctx->devices.size()) ? ctx->devices[idx] : nullptr;
}
int pb2_device_link_bodies(pb2_device_module_t* dev, const void* image, size_t bytes, int format, uint32_t sliceable) {
    if (!dev || !PB2_DEV_IS_GPU(dev->type)) return PB2_ERR_BAD_PARAM;
    pb2_context_t* ctx = dev->ctx;
    if (const char* why = link_args_error(image, bytes, format, sliceable)) { ctx->last_error = why; return PB2_ERR_BAD_PARAM; }
    if (dev->linked) { ctx->last_error = "the module has linked an image already (one per module)"; return PB2_ERR_EXISTS; }
    if (dev->st.windows_launched) { ctx->last_error = "linked bodies must be linked before the module's first window"; return PB2_ERR_NOT_SUPPORTED; }
    if (!dev->dry_run) {
        const int rc = pb2_engine_link_bodies(dev->engine, image, bytes, format, sliceable);
        if (rc != PB2_SUCCESS) { ctx->last_error = pb2_engine_last_error(dev->engine); return rc; }
    }
    dev->linked = true;
    return PB2_SUCCESS;
}

int pb2_device_get_stats(pb2_device_module_t* dev, pb2_device_stats_t* st) { if (!dev || !st) return PB2_ERR_BAD_PARAM; *st = dev->st; return PB2_SUCCESS; }
static void best_unit(uint64_t bytes, double* v, const char** unit) {       // parsec_compute_best_unit: 1024-based
    static const char* units[] = {"B", "KB", "MB", "GB", "TB", "PB"};
    double x = (double)bytes; int u = 0;
    while (x >= 1024.0 && u < 5) { x /= 1024.0; ++u; }
    *v = x; *unit = units[u];
}

int pb2_devices_statistics_string(pb2_context_t* ctx, char* buf, size_t cap) {
    if (!ctx) return PB2_ERR_BAD_PARAM;
    std::string out;
    char line[512];
    uint64_t total_tasks = 0;
    for (auto* d : ctx->devices) total_tasks += d->st.executed_tasks;
    out += "device statistics (bytes moved vs bytes the tasks required)\n";
    out += " dev | name         |    kernels |      % | required in | moved H2D   (%)    | moved D2D   (%)    | required out | written back (%)  | evictions | windows | released on device\n";
    struct Tot { uint64_t k = 0, rin = 0, h2d = 0, d2d = 0, rout = 0, out = 0, ev = 0, win = 0, rel = 0; } T;
    auto row = [&](const char* id, const char* name, uint64_t k, uint64_t rin, uint64_t h2d, uint64_t d2d, uint64_t rout, uint64_t o,
                   uint64_t ev, uint64_t win, uint64_t rel) {
        double a, b, c, e, f; const char *ua, *ub, *uc, *ue, *uf;
        best_unit(rin, &a, &ua); best_unit(h2d, &b, &ub); best_unit(d2d, &c, &uc); best_unit(rout, &e, &ue); best_unit(o, &f, &uf);
        snprintf(line, sizeof line, " %3s | %-12s | %10llu | %6.2f | %8.2f %-2s | %8.2f %-2s (%6.2f) | %8.2f %-2s (%6.2f) | %9.2f %-2s | %8.2f %-2s (%6.2f) | %9llu | %7llu | %llu\n",
                 id, name, (unsigned long long)k, total_tasks ? 100.0 * (double)k / (double)total_tasks : 0.0,
                 a, ua, b, ub, rin ? 100.0 * (double)h2d / (double)rin : 0.0, c, uc, rin ? 100.0 * (double)d2d / (double)rin : 0.0,
                 e, ue, f, uf, rout ? 100.0 * (double)o / (double)rout : 0.0,
                 (unsigned long long)ev, (unsigned long long)win, (unsigned long long)rel);
        out += line;
    };
    for (auto* d : ctx->devices) {
        uint64_t d2d = 0;
        for (int k = 2; k < PB2_MAX_DEVICES; ++k) d2d += d->st.data_in_from_device[k];
        char id[8]; snprintf(id, sizeof id, "%d", (int)d->device_index);
        row(id, d->name.c_str(), d->st.executed_tasks, d->st.required_data_in, d->st.data_in_from_device[0], d2d, d->st.required_data_out,
            d->st.data_out_to_host, d->st.nb_evictions, d->st.windows_launched, d->st.tasks_released_on_device);
        T.k += d->st.executed_tasks; T.rin += d->st.required_data_in; T.h2d += d->st.data_in_from_device[0]; T.d2d += d2d;
        T.rout += d->st.required_data_out; T.out += d->st.data_out_to_host; T.ev += d->st.nb_evictions;
        T.win += d->st.windows_launched; T.rel += d->st.tasks_released_on_device;
    }
    row("all", "", T.k, T.rin, T.h2d, T.d2d, T.rout, T.out, T.ev, T.win, T.rel);
    if (buf && cap) { const size_t n = out.size() < cap - 1 ? out.size() : cap - 1; memcpy(buf, out.data(), n); buf[n] = 0; }
    return (int)out.size() + 1;
}

int pb2_device_index(pb2_device_module_t* dev) { return dev ? dev->device_index : -1; }
int pb2_device_type(pb2_device_module_t* dev) { return dev ? dev->type : 0; }

void* pb2_device_zone_malloc(pb2_device_module_t* dev, size_t size) { return dev ? dev->zone.malloc(size) : nullptr; }
int pb2_device_zone_free(pb2_device_module_t* dev, void* ptr) { return dev ? dev->zone.free(ptr) : PB2_ERR_BAD_PARAM; }
size_t pb2_device_zone_in_use(pb2_device_module_t* dev) { return dev ? dev->zone.in_use() : 0; }
int pb2_device_lru_sizes(pb2_device_module_t* dev, int* clean, int* owned) {
    if (!dev) return PB2_ERR_BAD_PARAM;
    if (clean) *clean = dev->lru_count[1];
    if (owned) *owned = dev->lru_count[2];
    return PB2_SUCCESS;
}

int pb2_device_memory_register(pb2_device_module_t* dev, pb2_data_collection_t* dc, void* ptr, size_t len) {
    if (!dev || !ptr || !len) return PB2_ERR_BAD_PARAM;
    if (!PB2_DEV_IS_GPU(dev->type)) return PB2_SUCCESS;
    if (dc && (dc->memory_registration_status & (1u << dev->device_index))) return PB2_SUCCESS;   // idempotent (:189-193)
    void* alias = ptr;
    if (!dev->dry_run) {
        int rc = pb2_engine_host_register(dev->engine, ptr, len, &alias);
        if (rc != PB2_SUCCESS) return rc;
    }
    if (dc) { dc->memory_registration_status |= 1u << dev->device_index; dc->device_alias[dev->device_index] = alias; }
    else dev->host_alias[ptr] = alias;
    return PB2_SUCCESS;
}
int pb2_device_memory_unregister(pb2_device_module_t* dev, pb2_data_collection_t* dc, void* ptr) {
    if (!dev || !ptr) return PB2_ERR_BAD_PARAM;
    if (!PB2_DEV_IS_GPU(dev->type)) return PB2_SUCCESS;
    if (dc && !(dc->memory_registration_status & (1u << dev->device_index))) return PB2_SUCCESS;
    if (!dev->dry_run) pb2_engine_host_unregister(dev->engine, ptr);
    if (dc) { dc->memory_registration_status &= ~(1u << dev->device_index); dc->device_alias.erase(dev->device_index); }
    else dev->host_alias.erase(ptr);
    return PB2_SUCCESS;
}

int pb2_device_taskpool_register(pb2_device_module_t* dev, pb2_taskpool_t* tp) {
    // device_gpu.c:785-836: a taskpool keeps its device bit only if some chore of it can run on this device type
    if (!dev || !tp) return PB2_ERR_BAD_PARAM;
    bool any = false;
    for (auto& tc : tp->classes) if (tc.chore_types & dev->type) any = true;
    if (!any) { tp->devices_index_mask &= ~(1u << dev->device_index); return PB2_ERR_NOT_FOUND; }
    return PB2_SUCCESS;
}
int pb2_device_taskpool_unregister(pb2_device_module_t* dev, pb2_taskpool_t* tp) { (void)dev; (void)tp; return PB2_SUCCESS; }

}  // extern "C"

// device-visible address of a datum's host copy on `dev` (needs the memory to be registered / pinned)
void* pb2i_device_visible_host_ptr(pb2_device_module_t* dev, pb2_data_t* data) {
    pb2_data_copy_t* h = pb2i_host_copy(data);
    if (!h || !h->device_private) return nullptr;
    pb2_data_collection_t* dc = data->dc;
    if (dc && dc->mat) {
        if (!(dc->memory_registration_status & (1u << dev->device_index))) {
            // the PTG startup hook registers every collection (jdf2c.c:4501-4508); DTD users get it on first touch
            size_t len = (size_t)dc->nb_local_tiles * (size_t)dc->bsiz * (size_t)dc->elt_bytes;
            if (pb2_device_memory_register(dev, dc, dc->mat, len) != PB2_SUCCESS) return nullptr;
        }
        char* alias = reinterpret_cast<char*>(dc->device_alias[dev->device_index]);
        return alias + (reinterpret_cast<char*>(h->device_private) - reinterpret_cast<char*>(dc->mat));
    }
    auto it = dev->host_alias.find(h->device_private);
    if (it != dev->host_alias.end()) return it->second;
    if (pb2_device_memory_register(dev, nullptr, h->device_private, data->span ? data->span : 16) != PB2_SUCCESS) return nullptr;
    return dev->host_alias[h->device_private];
}

// =============================================================================================
// device selection (device.c:100-310) and task progress (scheduling.c)
// =============================================================================================
static int64_t time_estimate(pb2_htask_t* t, pb2_device_module_t* d) { (void)t; return d->st.time_estimate_default; }

extern "C" int pb2_select_best_device(pb2_context_t* ctx, pb2_htask_t* t) {
    pb2_taskpool_t* tp = t->tp;
    if (t->selected_device) return t->selected_device->device_index;
    const uint8_t valid_types = t->chore_types & t->allowed_types;
    if (!valid_types) return -1;
    auto usable = [&](int d) -> pb2_device_module_t* {
        if (d < 0 || d >= (int)ctx->devices.size()) return nullptr;
        pb2_device_module_t* dev = ctx->devices[d];
        return ((dev->type & valid_types) && (tp->devices_index_mask & (1u << d))) ? dev : nullptr;
    };
    if (valid_types == PB2_DEV_CPU) { t->selected_device = ctx->devices[0]; t->load = 0; return 0; }
    pb2_device_module_t* rdata_dev = nullptr;
    for (int i = 0; i < t->nb_flows; i++) {                        // first ACCESS_WRITE data (:170-192)
        if (!(t->access[i] & PB2_FLOW_ACCESS_WRITE) || !t->data[i]) continue;
        if (pb2_device_module_t* dev = usable(t->data[i]->preferred_device)) { t->selected_device = dev; goto selected; }
        pb2_device_module_t* dev = usable(t->data[i]->owner_device);
        if (dev && PB2_DEV_IS_GPU(dev->type)) { t->selected_device = dev; goto selected; }
    }
    for (int i = 0; i < t->nb_flows; i++) {                        // then READ data (:194-217)
        if (!(t->access[i] & PB2_FLOW_ACCESS_READ) || !t->data[i]) continue;
        if (pb2_device_module_t* dev = usable(t->data[i]->preferred_device)) { t->selected_device = dev; goto selected; }
        pb2_device_module_t* dev = usable(t->data[i]->owner_device);
        if (dev && PB2_DEV_IS_GPU(dev->type)) { rdata_dev = dev; break; }
    }
    {
        int best_index = -1;
        int64_t best_eta = INT64_MAX;
        const float skew = 1.f / ((float)ctx->mca["device_load_balance_skew"] / 100.f + 1.f);
        if (rdata_dev) {
            best_index = rdata_dev->device_index;
            best_eta = (int64_t)((float)(rdata_dev->st.device_load + time_estimate(t, rdata_dev)) * skew);
        }
        for (int d = (int)ctx->devices.size() - 1; d >= 0; d--) {
            pb2_device_module_t* dev = usable(d);
            if (!dev || (dev->type & PB2_DEV_RECURSIVE)) continue;
            const int64_t eta = dev->st.device_load + time_estimate(t, dev);
            if (best_eta > eta) {
                if (best_index != -1 && !PB2_DEV_IS_GPU(dev->type) && !ctx->mca["device_load_balance_allow_cpu"]) continue;
                best_index = d; best_eta = eta;
            }
        }
        if (best_index < 0) return -1;
        t->selected_device = ctx->devices[best_index];
    }
selected:
    t->load = time_estimate(t, t->selected_device);
    return t->selected_device->device_index;
}

// parsec_list_push_sorted by priority (higher first, FIFO among equals)
void pb2i_schedule(pb2_context_t* ctx, pb2_htask_t* t) {
    t->state = 1;
    auto it = ctx->ready.end();
    const auto first = ctx->ready.begin() + (long)ctx->ready_head;
    while (it != first && (*(it - 1))->priority < t->priority) --it;
    ctx->ready.insert(it, t);
}

pb2_htask_t* pb2i_new_task(pb2_taskpool_t* tp, pb2_task_class_t* tc) {
    tp->tasks.emplace_back();
    pb2_htask_t* t = &tp->tasks.back();
    t->tp = tp; t->tc = tc; t->id = (int32_t)tp->tasks.size() - 1;
    if (tc) { t->nb_flows = tc->nb_flows; t->use_mask = tc->use_mask; t->chore_types = tc->chore_types;
              t->body = tc->gpu_body >= 0 ? (uint8_t)tc->gpu_body : 0; }
    return t;
}

void pb2i_add_edge(pb2_taskpool_t* tp, int32_t src, int32_t dst, int dst_flow) {
    tp->tasks[src].succ.push_back(PB2_SUCC_MAKE(dst, dst_flow));
    pb2_htask_t& d = tp->tasks[dst];
    d.npred_unsat++;
    if (d.use_mask) d.dep_goal |= 1 << dst_flow; else { d.dep_goal++; d.dep_word++; }
}

// the predecessor's output copy becomes the successor's input (parsec.c:1800-1803, overlap_strategies.c:268)
static void forward_data(pb2_htask_t* pred, pb2_htask_t* t, int flow) {
    if (!t->data[flow]) return;
    for (int f = 0; f < pred->nb_flows; ++f)
        if (pred->data[f] == t->data[flow] && pred->data_out[f]) t->data_in[flow] = pred->data_out[f];
}

// host-side release of one out-edge: parsec_release_local_OUT_dependencies (parsec.c:1749-1834)
static void release_edge(pb2_context_t* ctx, pb2_htask_t* pred, uint32_t s) {
    pb2_taskpool_t* tp = pred->tp;
    pb2_htask_t* t = &tp->tasks[PB2_SUCC_TASK(s)];
    const int flow = PB2_SUCC_FLOW(s);
    t->npred_unsat--;
    bool ready;
    if (t->use_mask) { t->dep_word |= 1 << flow; ready = (t->dep_word & t->dep_goal) == t->dep_goal; }   // parsec.c:1656
    else ready = (--t->dep_word == 0);                                                                     // parsec.c:1609
    if (ready && t->state == 0) pb2i_schedule(ctx, t);
}

int pb2i_complete_execution(pb2_context_t* ctx, pb2_htask_t* t, int device_index) {
    t->state = 3; t->ran_on = (int8_t)device_index;
    pb2_taskpool_t* tp = t->tp;
    tp->trace_task.push_back(t->id); tp->trace_device.push_back(device_index);
    for (uint32_t s : t->succ) {
        pb2_htask_t* n = &tp->tasks[PB2_SUCC_TASK(s)];
        forward_data(t, n, PB2_SUCC_FLOW(s));
        if (n->window_index >= 0 || n->state >= 2) {
            // released by a device atomic inside the window: only keep the host dependency words in sync
            n->npred_unsat--;
            if (n->use_mask) n->dep_word |= 1 << PB2_SUCC_FLOW(s); else n->dep_word--;
            continue;
        }
        release_edge(ctx, t, s);
    }
    if (t->selected_device) t->selected_device->st.device_load -= t->load;     // scheduling.c:496
    tp->nb_done++;
    return PB2_SUCCESS;
}

// CPU incarnation: ensure the host copy is the valid one, run the hook, bump versions (scheduling.c:148-164)
static int run_cpu_task(pb2_context_t* ctx, pb2_htask_t* t) {
    void* ptrs[PB2_MAX_FLOWS] = {nullptr, nullptr, nullptr, nullptr};
    for (int f = 0; f < t->nb_flows; ++f) {
        pb2_data_t* d = t->data[f];
        if (!d) continue;
        pb2_data_copy_t* h = pb2i_host_copy(d);
        if (!h) return PB2_ERROR;
        // The newest version must be on the host before a CPU body reads it.  A producing GPU task normally pushed it
        // out; when it did not (no pushout requested, or an in-place write that left the coherency states untouched,
        // device_gpu.c:1832-1836) the decision is taken by VERSION, like every other one that moves bytes here: fetch
        // from the valid replica with the highest version whenever it is newer than the host copy.
        if (t->access[f] & PB2_FLOW_ACCESS_READ) {
            pb2_data_copy_t* newest = nullptr;
            for (int i = 2; i < (int)ctx->devices.size(); ++i) {
                pb2_data_copy_t* c = d->device_copies[i];
                if (c && c->device_private && c->coherency_state != PB2_DATA_COHERENCY_INVALID && c->version > h->version &&
                    (!newest || c->version > newest->version)) newest = c;
            }
            if (newest) {
                pb2_device_module_t* od = ctx->devices[newest->device_index];
                // the task that wrote this version has been retired (that is why this task is ready): the bytes are final;
                // the copy is ordered behind whatever the engine stream still runs
                if (!od->dry_run) { pb2_engine_memcpy_d2h(od->engine, h->device_private, newest->device_private, d->span); }
                od->st.data_out_to_host += d->span;
                h->version = newest->version;
                h->coherency_state = PB2_DATA_COHERENCY_SHARED; newest->coherency_state = PB2_DATA_COHERENCY_SHARED;
                d->owner_device = 0;
            }
        }
        pb2_data_start_transfer_ownership_to_copy(ctx, d, 0, t->access[f]);
        pb2_data_end_transfer_ownership_to_copy(d, 0, t->access[f]);
        t->seen_version[f] = h->version;
        t->data_in[f] = t->data_out[f] = h;
        ptrs[f] = h->device_private;
    }
    int rc = t->tc && t->tc->cpu_hook ? t->tc->cpu_hook(t, ptrs, t->iparam, t->fparam) : PB2_HOOK_RETURN_DONE;
    for (int f = 0; f < t->nb_flows; ++f) {
        pb2_data_t* d = t->data[f];
        if (!d) continue;
        pb2_data_copy_t* h = pb2i_host_copy(d);
        if (t->access[f] & PB2_FLOW_ACCESS_READ) h->readers--;
        if (t->access[f] & PB2_FLOW_ACCESS_WRITE) {
            // the CPU result supersedes EVERY replica, including GPU ones that are newer than the host copy was
            // (write-only flow after GPU writes without pushout): version = newest + 1, all the others stale
            uint32_t newest = h->version;
            for (int i = 1; i < PB2_MAX_DEVICES; ++i)
                if (d->device_copies[i] && d->device_copies[i]->version > newest) newest = d->device_copies[i]->version;
            h->version = newest + 1;
            h->coherency_state = PB2_DATA_COHERENCY_OWNED; d->owner_device = 0;
            for (int i = 1; i < PB2_MAX_DEVICES; ++i) {
                pb2_data_copy_t* c = d->device_copies[i];
                if (!c) continue;
                c->coherency_state = PB2_DATA_COHERENCY_INVALID;
                if (i >= 2 && c->lru_list == 2 && c->readers == 0) {          // nothing left to write back
                    pb2_device_module_t* od = ctx->devices[i];
                    pb2i_lru_remove(od, c); pb2i_lru_push_back(od, 1, c);
                }
            }
        }
    }
    ctx->devices[0]->st.executed_tasks++;
    return rc;
}

static int device_progress(pb2_device_module_t* dev);

// __parsec_execute + the generated GPU hook (jdf2c.c:6832-6969 / insert_function.c:2393-2425)
static int execute_task(pb2_context_t* ctx, pb2_htask_t* t) {
    const int d = pb2_select_best_device(ctx, t);
    if (d < 0) { ctx->last_error = "task ran out of valid incarnations"; return PB2_ERROR; }
    pb2_device_module_t* dev = ctx->devices[d];
    dev->st.device_load += t->load;                                 // scheduling.c:142
    if (!PB2_DEV_IS_GPU(dev->type)) {
        int rc = run_cpu_task(ctx, t);
        if (rc != PB2_HOOK_RETURN_DONE) { ctx->last_error = "CPU hook failed"; return PB2_ERROR; }
        return pb2i_complete_execution(ctx, t, 0);
    }
    pb2_gpu_task_t* g = new pb2_gpu_task_s();
    g->ec = t; g->task_type = 0; g->pushout = t->pushout; g->nb_flows = (uint32_t)t->nb_flows;
    for (int f = 0; f < t->nb_flows; ++f) g->flow_span[f] = t->data[f] ? t->data[f]->span : 0;
    const pb2_hook_return_t rc = pb2_device_kernel_scheduler(dev, nullptr, g);
    return rc == PB2_HOOK_RETURN_ASYNC ? PB2_SUCCESS : PB2_ERROR;   // anything else is fatal (scheduling.c:541-548)
}

extern "C" {

pb2_hook_return_t pb2_device_kernel_scheduler(pb2_device_module_t* dev, void* es, void* gpu_task) {
    (void)es;
    if (!dev || !gpu_task || !PB2_DEV_IS_GPU(dev->type)) return PB2_HOOK_RETURN_DISABLE;
    pb2_gpu_task_t* g = reinterpret_cast<pb2_gpu_task_t*>(gpu_task);
    g->ec->state = 2;
    dev->pending.push_back(g);                                      // parsec_fifo_push(&gpu_device->pending)
    dev->mutex++;
    return PB2_HOOK_RETURN_ASYNC;                                   // the device owns the task from here on
}

int pb2_context_add_taskpool(pb2_context_t* ctx, pb2_taskpool_t* tp) {
    if (!ctx || !tp) return PB2_ERR_BAD_PARAM;
    if (!tp->added) { ctx->taskpools.push_back(tp); tp->added = true; }
    for (auto* d : ctx->devices) if (PB2_DEV_IS_GPU(d->type)) pb2_device_taskpool_register(d, tp);
    return PB2_SUCCESS;
}
int pb2_context_start(pb2_context_t* ctx) { if (!ctx) return PB2_ERR_BAD_PARAM; ctx->started = true; return PB2_SUCCESS; }

int pb2_context_wait(pb2_context_t* ctx) {
    if (!ctx) return PB2_ERR_BAD_PARAM;
    if (!ctx->devices_frozen) pb2_mca_device_registration_complete(ctx);
    for (;;) {
        bool progressed = false;
        const double t_sched = now_ms();
        const size_t nready0 = ctx->ready.size();
        // pop from the front without shifting the vector each time: ready_head marks what has been taken, and
        // pb2i_schedule never inserts in front of it
        while (ctx->ready_head < ctx->ready.size()) {
            pb2_htask_t* t = ctx->ready[ctx->ready_head++];
            int rc = execute_task(ctx, t);
            if (rc != PB2_SUCCESS) { ctx->ready.erase(ctx->ready.begin(), ctx->ready.begin() + (long)ctx->ready_head); ctx->ready_head = 0; return rc; }
            progressed = true;
        }
        ctx->ready.clear(); ctx->ready_head = 0;
        if (g_timing && nready0) fprintf(stderr, "pb2 wait: dispatched %zu ready tasks in %.2f ms\n", nready0, now_ms() - t_sched);
        for (auto* d : ctx->devices) {
            if (!PB2_DEV_IS_GPU(d->type) || (d->pending.empty() && d->inflight.empty())) continue;
            int rc = device_progress(d);
            if (rc != PB2_SUCCESS) return rc;
            progressed = true;
        }
        bool all_done = true;
        for (auto* tp : ctx->taskpools) if (tp->nb_done != (int32_t)tp->tasks.size()) all_done = false;
        if (all_done) break;
        if (!progressed) { ctx->last_error = "deadlock: tasks left but nothing is ready"; return PB2_ERROR; }
    }
    for (auto* tp : ctx->taskpools) if (tp->on_complete) { auto f = tp->on_complete; tp->on_complete = nullptr; f(); }
    ctx->started = false;
    return PB2_SUCCESS;
}

int pb2_taskpool_wait(pb2_taskpool_t* tp) { return tp ? pb2_context_wait(tp->ctx) : PB2_ERR_BAD_PARAM; }
int pb2_taskpool_nb_tasks(pb2_taskpool_t* tp) { return tp ? (int)tp->tasks.size() : 0; }
int pb2_taskpool_set_device_types(pb2_taskpool_t* tp, int types) {
    if (!tp) return PB2_ERR_BAD_PARAM;
    for (size_t i = 0; i < tp->tasks.size(); ++i) { pb2_htask_t& t = tp->tasks[i]; t.allowed_types = (uint8_t)types; t.selected_device = nullptr; }
    return PB2_SUCCESS;
}

int pb2_taskpool_completion_trace(pb2_taskpool_t* tp, int32_t* out_task, int32_t* out_device, int32_t cap) {
    if (!tp) return PB2_ERR_BAD_PARAM;
    const int32_t n = (int32_t)tp->trace_task.size();
    for (int32_t i = 0; i < n && i < cap; ++i) { if (out_task) out_task[i] = tp->trace_task[i]; if (out_device) out_device[i] = tp->trace_device[i]; }
    return n;
}

int pb2_taskpool_device_trace(pb2_taskpool_t* tp, uint64_t* t_start_ns, uint64_t* t_end_ns, int32_t* device, uint32_t* smid) {
    if (!tp) return PB2_ERR_BAD_PARAM;
    for (size_t i = 0; i < tp->tasks.size(); ++i) {
        const pb2_htask_s& t = tp->tasks[i];
        if (t_start_ns) t_start_ns[i] = t.dev_t_start;
        if (t_end_ns) t_end_ns[i] = t.dev_t_end;
        if (device) device[i] = t.ran_on;
        if (smid) smid[i] = t.dev_smid;
    }
    return PB2_SUCCESS;
}

int pb2_taskpool_device_part_trace(pb2_taskpool_t* tp, pb2_part_trace_t* out, int32_t* device, int32_t cap, int32_t* n) {
    if (!tp || !n || cap < 0) return PB2_ERR_BAD_PARAM;
    const int32_t total = (int32_t)tp->part_trace.size();
    *n = total;
    for (int32_t i = 0; i < total && i < cap; ++i) {
        if (out) out[i] = tp->part_trace[(size_t)i];
        if (device) device[i] = tp->part_trace_device[(size_t)i];
    }
    return PB2_SUCCESS;
}

int pb2_taskpool_task_info(pb2_taskpool_t* tp, int32_t* class_id, int32_t* locals2, uint32_t* seen_version4, uint64_t* result) {
    if (!tp) return PB2_ERR_BAD_PARAM;
    for (size_t i = 0; i < tp->tasks.size(); ++i) {
        const pb2_htask_s& t = tp->tasks[i];
        if (class_id) class_id[i] = t.tc ? t.tc->task_class_id : -1;
        if (locals2) { locals2[2 * i] = t.locals[0]; locals2[2 * i + 1] = t.locals[1]; }
        if (seen_version4) for (int f = 0; f < 4; ++f) seen_version4[4 * i + f] = t.seen_version[f];
        if (result) result[i] = t.result;
    }
    return PB2_SUCCESS;
}

int pb2_taskpool_free(pb2_taskpool_t* tp) {
    if (!tp) return PB2_ERR_BAD_PARAM;
    pb2_context_t* ctx = tp->ctx;
    ctx->taskpools.erase(std::remove(ctx->taskpools.begin(), ctx->taskpools.end(), tp), ctx->taskpools.end());
    for (auto* t : tp->tile_list) delete t;
    for (pb2_data_t* d : tp->temporaries) {
        for (auto* dev : ctx->devices) {
            pb2_data_copy_t* c = d->device_copies[dev->device_index];
            if (c && dev->device_index >= 2) { pb2i_lru_remove(dev, c); if (c->device_private) dev->zone.free(c->device_private); }
        }
        data_destroy(d);
    }
    delete tp;
    return PB2_SUCCESS;
}

}  // extern "C"

// =============================================================================================
// the GPU device module: window building, launch, retire
// =============================================================================================

// Write back up to max_copies dirty replicas (transfer_gpu.c:224-362, with the intended outcome: the host copy
// gets the replica's version, both become SHARED, the replica moves to the clean LRU).  All the copies of one
// call travel in ONE kernel launch (pb2_engine_copy_batch) instead of one cudaMemcpyAsync + event per tile.
static int w2r_flush(pb2_device_module_t* dev, int max_copies) {
    std::vector<pb2_data_copy_t*> picked, stale;
    std::vector<void*> dst; std::vector<const void*> src; std::vector<uint64_t> bytes;
    for (pb2_data_copy_t* c = dev->lru_head[2]; c && (int)picked.size() < max_copies; c = c->lru_next) {
        pb2_data_t* d = c->original;
        pb2_data_copy_t* h = pb2i_host_copy(d);
        if (c->readers != 0 || c->window_tile >= 0 || !h || !h->device_private) continue;
        if (c->version <= h->version) { stale.push_back(c); continue; }   // another device wrote the tile home since: nothing to save
        void* alias = dev->dry_run ? h->device_private : pb2i_device_visible_host_ptr(dev, d);
        if (!alias) continue;
        picked.push_back(c); dst.push_back(alias); src.push_back(c->device_private); bytes.push_back(d->span);
    }
    for (pb2_data_copy_t* c : stale) pb2i_lru_push_back(dev, 1, c);      // not dirty any more: plain eviction candidates
    if (picked.empty()) return (int)stale.size();
    if (!dev->dry_run) {
        if (pb2_engine_copy_batch(dev->engine, dst.data(), src.data(), bytes.data(), (int32_t)picked.size()) != PB2_SUCCESS) return 0;
        pb2_engine_synchronize(dev->engine);
    }
    for (pb2_data_copy_t* c : picked) {
        pb2_data_t* d = c->original;
        pb2_data_copy_t* h = pb2i_host_copy(d);
        dev->st.data_out_to_host += d->span;
        c->coherency_state = PB2_DATA_COHERENCY_SHARED; h->coherency_state = PB2_DATA_COHERENCY_SHARED;
        h->version = c->version; h->flags |= PB2_DATA_FLAG_EVICTED;
        if (d->owner_device == dev->device_index) d->owner_device = -1;
        pb2i_lru_push_back(dev, 1, c);
    }
    return (int)(picked.size() + stale.size());
}

// Evict one clean replica not used by the window under construction (reserve_space :1339-1575)
static bool evict_one(pb2_device_module_t* dev) {
    for (pb2_data_copy_t* c = dev->lru_head[1]; c; c = c->lru_next) {
        if (c->readers != 0 || c->window_tile >= 0) continue;
        pb2_data_t* d = c->original;
        { const pb2_data_copy_t* h = pb2i_host_copy(d); if (!h || c->version > h->version) continue; }   // never drop the only newest version
        pb2i_lru_remove(dev, c);
        dev->zone.free(c->device_private);
        // The replica object stays attached to its datum, without a slot and INVALID: completed tasks still name it as
        // their output (data_out) and later consumers as their input (data_in); the reference keeps such objects alive
        // by reference counting (PARSEC_OBJ_RETAIN in the repo entries).  reserve_space gives it a slot again.
        c->device_private = nullptr;
        c->coherency_state = PB2_DATA_COHERENCY_INVALID; c->version = 0; c->readers = 0;
        c->data_transfer_status = PB2_DATA_STATUS_NOT_TRANSFER;
        if (d->owner_device == dev->device_index) d->owner_device = -1;
        dev->st.nb_evictions++;
        return true;
    }
    return false;
}

// parsec_device_data_reserve_space for one datum: find or create the replica, give it an HBM slot
static pb2_data_copy_t* reserve_space(pb2_device_module_t* dev, pb2_data_t* d) {
    pb2_data_copy_t* g = d->device_copies[dev->device_index];
    if (g && g->device_private) return g;
    void* slot = nullptr;
    for (;;) {
        slot = dev->zone.malloc(d->span ? d->span : 1);
        if (slot) break;
        if (evict_one(dev)) continue;
        if (w2r_flush(dev, (int)dev->ctx->mca["device_cuda_max_number_of_ejected_data"]) > 0) continue;
        return nullptr;                                             // PARSEC_HOOK_RETURN_AGAIN
    }
    if (!g) g = new_copy(d, dev->device_index, PB2_DATA_FLAG_PARSEC_OWNED | PB2_DATA_FLAG_PARSEC_MANAGED);
    g->device_private = slot;
    g->coherency_state = PB2_DATA_COHERENCY_INVALID; g->version = 0; g->readers = 0;
    g->data_transfer_status = PB2_DATA_STATUS_NOT_TRANSFER;
    return g;
}

// where would the bytes come from if this replica had to be filled now (stage_in source choice :1888-2008)
static pb2_data_copy_t* stage_in_source(pb2_device_module_t* dev, pb2_data_t* d) {
    pb2_context_t* ctx = dev->ctx;
    uint32_t newest = 0;
    for (size_t i = 0; i < ctx->devices.size(); ++i)
        if (d->device_copies[i] && d->device_copies[i]->coherency_state != PB2_DATA_COHERENCY_INVALID && d->device_copies[i]->version > newest)
            newest = d->device_copies[i]->version;
    for (size_t i = 2; i < ctx->devices.size(); ++i) {              // a peer GPU replica of the newest version first
        pb2_data_copy_t* c = d->device_copies[i];
        if ((int)i == dev->device_index || !c || !c->device_private) continue;
        if (!(dev->peer_access_mask & (1u << i))) continue;
        if (c->coherency_state != PB2_DATA_COHERENCY_INVALID && c->version == newest &&
            c->data_transfer_status != PB2_DATA_STATUS_UNDER_TRANSFER) return c;
    }
    return pb2i_host_copy(d);
}

struct Window {
    pb2_taskpool_t* tp = nullptr;
    std::vector<pb2_htask_t*> order;
    std::vector<pb2_data_t*> tile_data;
    std::vector<pb2_tile_t> tiles;
    std::vector<pb2_data_copy_t*> tile_src;
    std::vector<uint8_t> tile_staged;       // the window moves this tile in for its first reader (decided at build, by version)
    std::vector<pb2_data_copy_t*> src_held; // peer replicas pinned (readers++) as stage-in sources until the window retires
    std::vector<pb2_task_t> tasks;
    std::vector<uint32_t> succ;
    std::vector<int32_t> ready;
    int kind = 0;
};

static bool predicted_on_device(pb2_device_module_t* dev, pb2_htask_t* s) {
    if (!((s->chore_types & s->allowed_types) & PB2_DEV_CUDA)) return false;
    if (!(s->tp->devices_index_mask & (1u << dev->device_index))) return false;
    for (int f = 0; f < s->nb_flows; ++f) {
        if (!(s->access[f] & PB2_FLOW_ACCESS_WRITE) || !s->data[f]) continue;
        const int p = s->data[f]->preferred_device;
        if (p >= 0) return p == dev->device_index;
        break;
    }
    for (int f = 0; f < s->nb_flows; ++f) {
        if (!s->data[f]) continue;
        const int p = s->data[f]->preferred_device;
        if (p >= 0) return p == dev->device_index;
    }
    return true;   // no affinity: stays with its predecessor's device
}

// Build the dependency-closed window reachable from the pending tasks of one taskpool.  An engine window takes tile
// GEMMs and HBM bodies together, so that a GEMM chain and the element-wise tasks around it are released on the device
// instead of through the host; its kind is decided by the closure: 1 (the GEMM kernel, which also runs HBM bodies) when
// it holds a GEMM task, else 0.  User submit tasks never mix with engine tasks, and tasks of linked bodies (which run in
// the linked HBM kernel only) never mix with GEMM tasks: the first of the two kinds the closure takes in keeps the other
// out of this window.
static int build_window(pb2_device_module_t* dev, Window& w, std::vector<pb2_gpu_task_t*>& taken, size_t max_roots) {
    if (dev->pending.empty()) return PB2_SUCCESS;
    w.tp = dev->pending.front()->ec->tp;
    const bool want_user = dev->pending.front()->ec->body == PB2_BODY_USER;      // the host-driven stream lane
    int engine_side = 0;                        // PB2_BODY_GEMM_BF16 or PB2_BODY_LINKED_0 once the window holds one
    auto fits = [&](const pb2_htask_t* t) {
        if ((t->body == PB2_BODY_USER) != want_user) return false;
        const int side = t->body == PB2_BODY_GEMM_BF16 ? PB2_BODY_GEMM_BF16 : pb2::is_linked_body(t->body) ? PB2_BODY_LINKED_0 : 0;
        if (side && engine_side && side != engine_side) return false;
        if (side) engine_side = side;
        return true;
    };
    bool has_gemm = false;
    std::deque<pb2_htask_t*> queue;
    std::deque<pb2_gpu_task_t*> keep;
    for (pb2_gpu_task_t* g : dev->pending) {
        if (taken.size() < max_roots && g->ec->tp == w.tp && fits(g->ec)) { queue.push_back(g->ec); taken.push_back(g); }
        else keep.push_back(g);
    }
    dev->pending.swap(keep);
    std::vector<pb2_htask_t*> touched;
    bool full = false;
    while (!queue.empty()) {
        pb2_htask_t* t = queue.front(); queue.pop_front();
        // the ready-ring entries of an HBM window carry a 22-bit task id: a larger closure without a GEMM task (which
        // would make it a GEMM window, whose entries carry 27-bit unit ids) goes on in the next window
        if (!want_user && !has_gemm && w.order.size() + 1 >= ((size_t)1 << 22)) full = true;
        bool ok = !full;
        std::vector<pb2_data_copy_t*> fresh;
        if (ok) {
            for (int f = 0; f < t->nb_flows && ok; ++f) {           // kernel_push: reserve_space per flow
                pb2_data_t* d = t->data[f];
                if (!d) continue;
                pb2_data_copy_t* g = reserve_space(dev, d);
                if (!g) { ok = false; break; }
                if (g->window_tile >= 0 && g->window_owner != &w) { ok = false; break; }   // in use by the window that is running
                if (g->window_tile < 0) {
                    g->window_tile = (int32_t)w.tile_data.size();
                    g->window_owner = &w;
                    w.tile_data.push_back(d);
                    fresh.push_back(g);
                }
            }
        }
        if (!ok) {
            // no room: this task (and everything behind it) waits for the next window (HOOK_RETURN_AGAIN)
            full = true;
            for (pb2_data_copy_t* g : fresh) {
                g->window_tile = -1; g->window_owner = nullptr; w.tile_data.pop_back();
                // a slot reserve_space has just allocated for this task is on no list yet: put it where eviction finds it
                if (g->lru_list == 0) pb2i_lru_push_back(dev, (g->coherency_state == PB2_DATA_COHERENCY_OWNED && g->version > 0) ? 2 : 1, g);
            }
            continue;
        }
        t->window_index = (int32_t)w.order.size();
        w.order.push_back(t);
        has_gemm |= t->body == PB2_BODY_GEMM_BF16;
        for (uint32_t s : t->succ) {
            pb2_htask_t* n = &w.tp->tasks[PB2_SUCC_TASK(s)];
            if (n->inwin_pred == 0) touched.push_back(n);
            n->inwin_pred++;
            if (n->state == 0 && n->inwin_pred == n->npred_unsat && predicted_on_device(dev, n) && fits(n))
                queue.push_back(n);
        }
    }
    for (pb2_htask_t* n : touched) n->inwin_pred = 0;
    w.kind = want_user ? 2 : (has_gemm ? 1 : 0);
    if (full) {      // tasks that were handed over but did not fit stay pending, in their arrival order
        std::vector<pb2_gpu_task_t*> in;
        for (pb2_gpu_task_t* g : taken) { if (g->ec->window_index >= 0) in.push_back(g); else dev->pending.push_back(g); }
        taken.swap(in);
    }
    if (w.order.empty()) {
        if (!dev->inflight.empty()) return PB2_SUCCESS;             // everything waits for the window that is running
        dev->ctx->last_error = "device memory too small for a single task"; return PB2_ERR_OUT_OF_RESOURCE;
    }

    // ---- tiles
    w.tiles.resize(w.tile_data.size());
    w.tile_src.assign(w.tile_data.size(), nullptr);
    for (size_t i = 0; i < w.tile_data.size(); ++i) {
        pb2_data_t* d = w.tile_data[i];
        pb2_data_copy_t* g = d->device_copies[dev->device_index];
        pb2i_lru_remove(dev, g);                                    // in use: off the lists until retire
        pb2_tile_t& tl = w.tiles[i];
        memset(&tl, 0, sizeof tl);
        tl.dev_ptr = g->device_private;
        if (d->span > 0xffffffffull) { dev->ctx->last_error = "tile larger than 4 GiB (pb2_tile_t::bytes is 32-bit)"; return PB2_ERR_VALUE_OUT_OF_BOUNDS; }
        tl.bytes = (uint32_t)d->span;
        uint32_t newest = 0;
        for (int k = 0; k < PB2_MAX_DEVICES; ++k)
            if (d->device_copies[k] && d->device_copies[k]->coherency_state != PB2_DATA_COHERENCY_INVALID && d->device_copies[k]->version > newest) newest = d->device_copies[k]->version;
        const bool valid_here = g->coherency_state != PB2_DATA_COHERENCY_INVALID && g->version >= newest;
        pb2_data_copy_t* src = valid_here ? nullptr : stage_in_source(dev, d);
        w.tile_src[i] = src;
        // a peer GPU's replica that this window will read from must stay where it is until the window has retired: hold
        // a reader on it, like the reference does for D2D sources (device_gpu.c:1925-1975, released :2461-2526)
        if (src && src->device_index >= 2 && src->device_index != dev->device_index) { src->readers++; w.src_held.push_back(src); }
        pb2_data_copy_t* h = pb2i_host_copy(d);
        const bool is_new = (d->dc == nullptr) && h && h->version == 0 && newest == 0;   // NEW: nothing to pull (:2049)
        if (valid_here) { tl.state = PB2_TILE_VALID; tl.version = g->version; }
        else if (is_new) { tl.state = PB2_TILE_VALID; tl.version = 0; w.tile_src[i] = nullptr; }
        else { tl.state = PB2_TILE_INVALID; tl.version = src ? src->version : 0; }
        w.tile_staged.push_back(tl.state == PB2_TILE_INVALID && src != nullptr);
        tl.src_kind = (src && src->device_index >= 2) ? PB2_SRC_PEER : PB2_SRC_HOST;
        // the home of the tile for pushout is always the host copy; a peer source is only used for stage-in
        void* host_alias = dev->dry_run ? (h ? h->device_private : nullptr) : pb2i_device_visible_host_ptr(dev, d);
        tl.src_ptr = (tl.src_kind == PB2_SRC_PEER) ? src->device_private : host_alias;
    }

    // ---- tasks + CSR of the in-window edges
    w.tasks.resize(w.order.size());
    for (size_t i = 0; i < w.order.size(); ++i) {
        pb2_htask_t* t = w.order[i];
        pb2_task_t& o = w.tasks[i];
        memset(&o, 0, sizeof o);
        o.priority = t->priority; o.body = t->body; o.nb_flows = (uint8_t)t->nb_flows;
        o.flags = t->use_mask ? PB2_TASK_DEPS_MASK : 0;
        o.class_id = t->tc ? (uint8_t)t->tc->task_class_id : 0;
        o.dep_goal = t->use_mask ? (t->dep_goal & ~t->dep_word) : t->dep_word;   // what is still missing
        for (int f = 0; f < PB2_MAX_FLOWS; ++f) {
            o.tile[f] = (f < t->nb_flows && t->data[f]) ? t->data[f]->device_copies[dev->device_index]->window_tile : -1;
            o.access[f] = f < t->nb_flows ? t->access[f] : 0;
            if (f < t->nb_flows && (t->pushout & (1 << f)) && t->data[f]) {
                const pb2_tile_t& tl = w.tiles[o.tile[f]];
                if (tl.src_kind == PB2_SRC_HOST && tl.src_ptr) o.access[f] |= PB2_FLOW_PUSHOUT;   // else host-side D2H at retire
            }
        }
        o.iparam[0] = t->iparam[0]; o.iparam[1] = t->iparam[1]; o.iparam[2] = t->iparam[2]; o.fparam = t->fparam;
        o.locals[0] = t->locals[0]; o.locals[1] = t->locals[1];
        o.succ_begin = (int32_t)w.succ.size();
        for (uint32_t s : t->succ) {
            pb2_htask_t* n = &w.tp->tasks[PB2_SUCC_TASK(s)];
            if (n->window_index >= 0) w.succ.push_back(PB2_SUCC_MAKE(n->window_index, PB2_SUCC_FLOW(s)));
        }
        o.succ_count = (int32_t)w.succ.size() - o.succ_begin;
        if (t->state == 2) w.ready.push_back((int32_t)i);          // handed over by kernel_scheduler: ready now
    }
    return PB2_SUCCESS;
}

static void window_release(pb2_device_module_t* dev, Window& w) {
    for (pb2_data_copy_t* c : w.src_held) c->readers--;
    w.src_held.clear();
    for (pb2_htask_t* t : w.order) t->window_index = -1;
    for (pb2_data_t* d : w.tile_data) if (d->device_copies[dev->device_index]) {
        d->device_copies[dev->device_index]->window_tile = -1; d->device_copies[dev->device_index]->window_owner = nullptr;
    }
}

// Host-visible bookkeeping of one retired task, replayed in retire order exactly as the reference's manager
// thread would have done it around the task: stage_in (device_gpu.c:1799-2165) + callback_complete_push
// (:2358-2573) for every flow, then kernel_pop (:2943-3173) + kernel_epilog (:3179-3292).
static void retire_task_bookkeeping(pb2_device_module_t* dev, Window& w, pb2_htask_t* t, const uint32_t* seen, uint64_t result) {
    pb2_context_t* ctx = dev->ctx;
    const int di = dev->device_index;
    for (int f = 0; f < t->nb_flows; ++f) {
        pb2_data_t* d = t->data[f];
        t->seen_version[f] = seen[f];
        if (!d) continue;
        pb2_data_copy_t* g = d->device_copies[di];
        const uint8_t acc = t->access[f];
        pb2_data_copy_t* in = t->data_in[f] ? t->data_in[f] : pb2i_host_copy(d);
        // the copy the task was given as input may have been evicted (and written back) since: the bytes then came from
        // the source chosen when the window was built (stage_in_source: newest valid replica, normally the host copy)
        if (in->coherency_state == PB2_DATA_COHERENCY_INVALID && in->device_index >= 2) {
            pb2_data_copy_t* src = w.tile_src[g->window_tile];
            in = src ? src : pb2i_host_copy(d);
        }
        dev->st.required_data_in += d->span;                                          // :2055
        if (in == g) {
            // "data already located in the right place" (:1820-1843): no ownership call at all
            if (acc & PB2_FLOW_ACCESS_WRITE) {
                // in-place write: this replica is now THE valid one -- say so in the protocol's own terms, so that
                // nobody (CPU bodies, other GPUs, the write-back) has to infer it from the version alone
                g->version++;
                g->coherency_state = PB2_DATA_COHERENCY_OWNED; d->owner_device = (int8_t)di;
                for (int i = 0; i < PB2_MAX_DEVICES; ++i)
                    if (i != di && d->device_copies[i] && d->device_copies[i]->coherency_state != PB2_DATA_COHERENCY_INVALID)
                        d->device_copies[i]->coherency_state = PB2_DATA_COHERENCY_SHARED;
            }
            if (acc & PB2_FLOW_ACCESS_READ) g->readers++;
        } else {
            // read-only flows may have been given a peer replica as source at build time (:1888-2008)
            pb2_data_copy_t* cand = (!(acc & PB2_FLOW_ACCESS_WRITE) && w.tile_src[g->window_tile]) ? w.tile_src[g->window_tile] : in;
            int from = pb2_data_start_transfer_ownership_to_copy(ctx, d, (uint8_t)di, acc);
            if (d->dc == nullptr && in->device_index == 0 && in->version == 0) from = -1;   // NEW, untouched (:2049-2052)
            // The window decided by VERSION whether this replica had to be refreshed (build_window: valid_here) and the
            // kernel moved the bytes for the first reader.  The coherency states alone can say "no transfer": a write to a
            // replica that is already in place leaves the other GPUs' older replicas SHARED (:1832-1836).  The replay
            // follows what was done.
            if ((acc & PB2_FLOW_ACCESS_READ) && w.tile_staged[(size_t)g->window_tile]) {
                w.tile_staged[(size_t)g->window_tile] = 0;
                if (w.tile_src[g->window_tile]) cand = w.tile_src[g->window_tile];
                if (from == -1 && !(d->dc == nullptr && cand->device_index == 0 && cand->version == 0)) {
                    from = cand->device_index;
                    g->coherency_state = PB2_DATA_COHERENCY_INVALID;
                }
            }
            if (from == -1) {
                g->data_transfer_status = PB2_DATA_STATUS_COMPLETE_TRANSFER;
                pb2_data_end_transfer_ownership_to_copy(d, (uint8_t)di, acc);
                if (acc & PB2_FLOW_ACCESS_WRITE) g->version = cand->version + 1;
            } else {
                dev->st.data_in_from_device[cand->device_index] += d->span;           // :2133
                dev->st.nb_data_faults += d->span;
                g->version = cand->version + ((acc & PB2_FLOW_ACCESS_WRITE) ? 1 : 0); // :2148-2152
                g->data_transfer_status = PB2_DATA_STATUS_COMPLETE_TRANSFER;           // callback_complete_push
                pb2_data_end_transfer_ownership_to_copy(d, (uint8_t)di, acc);
            }
        }
        t->data_in[f] = g; t->data_out[f] = g;
    }
    for (int f = 0; f < t->nb_flows; ++f) {                                            // pop + epilog
        pb2_data_t* d = t->data[f];
        if (!d) continue;
        pb2_data_copy_t* g = d->device_copies[di];
        const uint8_t acc = t->access[f];
        if (acc & PB2_FLOW_ACCESS_READ) g->readers--;
        if (!(acc & PB2_FLOW_ACCESS_WRITE)) continue;
        dev->st.required_data_out += d->span;                                          // :3078
        pb2_data_copy_t* h = pb2i_host_copy(d);
        if ((t->pushout & (1 << f)) && h) {
            const pb2_tile_t& tl = w.tiles[g->window_tile];
            if (!(tl.src_kind == PB2_SRC_HOST && tl.src_ptr) && !dev->dry_run && h->device_private)
                pb2_engine_memcpy_d2h(dev->engine, h->device_private, g->device_private, d->span);   // kernel could not
            dev->st.data_out_to_host += d->span;                                       // :3128
            h->version = g->version; h->coherency_state = PB2_DATA_COHERENCY_SHARED;   // epilog :3247-3255
            g->coherency_state = PB2_DATA_COHERENCY_SHARED;
            h->data_transfer_status = PB2_DATA_STATUS_COMPLETE_TRANSFER;
            t->data_out[f] = h;               // no GPU-aware sends: the host copy is the task's output (:3261-3274)
        }
    }
    t->result = result;
    dev->st.executed_tasks++;
}

struct InFlight {
    Window w;
    std::vector<pb2_gpu_task_t*> taken;
    pb2_window_t* win = nullptr;
    std::vector<uint32_t> lane_seen;        // kind 2 (user submit lane): versions seen, filled when the lane ran
    double t_begin = 0, t_built = 0, t_launched = 0;
};

// Tasks whose CUDA chore is a user `submit` function (PB2_BODY_USER): the host does for them what the reference's
// manager does for every task -- stage the inputs in (kernel_push), call submit on the stream (kernel_exec,
// device_gpu.c:2873-2934), write pushout flows back (kernel_pop) -- but for a whole dependency-closed chain of
// them at once and with batched copies: one copy kernel for all stage-ins, one for all write-backs.
static int run_submit_lane(pb2_device_module_t* dev, InFlight* f) {
    pb2_context_t* ctx = dev->ctx;
    Window& w = f->w;
    const size_t n = w.order.size();
    std::vector<void*> dst; std::vector<const void*> src; std::vector<uint64_t> len;
    std::vector<int8_t> first(w.tiles.size(), -1);
    for (size_t i = 0; i < n; ++i)
        for (int fl = 0; fl < w.tasks[i].nb_flows; ++fl) {
            const int32_t tile = w.tasks[i].tile[fl];
            if (tile >= 0 && first[(size_t)tile] < 0) first[(size_t)tile] = (w.tasks[i].access[fl] & PB2_FLOW_ACCESS_READ) ? 1 : 0;
        }
    for (size_t i = 0; i < w.tiles.size(); ++i) {
        const pb2_tile_t& tl = w.tiles[i];
        if (tl.state != PB2_TILE_INVALID || first[i] != 1 || !tl.src_ptr) continue;
        dst.push_back(tl.dev_ptr); src.push_back(tl.src_ptr); len.push_back(tl.bytes);
    }
    int rc = pb2_engine_copy_batch(dev->engine, dst.data(), src.data(), len.data(), (int32_t)dst.size());
    if (rc != PB2_SUCCESS) { ctx->last_error = std::string("submit lane stage-in: ") + pb2_engine_last_error(dev->engine); return rc; }
    void* stream = pb2_engine_get_stream(dev->engine);
    std::vector<uint32_t> ver(w.tiles.size());
    for (size_t i = 0; i < w.tiles.size(); ++i) ver[i] = w.tiles[i].version;
    f->lane_seen.assign(n * PB2_MAX_FLOWS, 0);
    dst.clear(); src.clear(); len.clear();
    for (size_t i = 0; i < n; ++i) {
        pb2_htask_t* t = w.order[i];
        if (!t->tc || !t->tc->submit) { ctx->last_error = "PB2_BODY_USER task without a submit function"; return PB2_ERR_BAD_PARAM; }
        pb2_gpu_task_s g;
        g.ec = t; g.pushout = t->pushout; g.nb_flows = (uint32_t)t->nb_flows;
        for (int fl = 0; fl < t->nb_flows; ++fl) g.flow_span[fl] = t->data[fl] ? t->data[fl]->span : 0;
        int hr = t->tc->submit(dev, &g, stream);
        for (int again = 0; hr == PB2_HOOK_RETURN_AGAIN && again < 1000; ++again) {      // device_gpu.c:2634-2641
            pb2_engine_synchronize(dev->engine);
            hr = t->tc->submit(dev, &g, stream);
        }
        if (hr != PB2_HOOK_RETURN_DONE && hr != PB2_HOOK_RETURN_ASYNC) { ctx->last_error = "submit function failed"; return PB2_ERROR; }
        for (int fl = 0; fl < t->nb_flows; ++fl) {
            const int32_t tile = w.tasks[i].tile[fl];
            if (tile < 0) continue;
            f->lane_seen[i * PB2_MAX_FLOWS + (size_t)fl] = ver[(size_t)tile];
            if (w.tasks[i].access[fl] & PB2_FLOW_ACCESS_WRITE) {
                ver[(size_t)tile]++;
                if (w.tasks[i].access[fl] & PB2_FLOW_PUSHOUT) {        // newest version goes home; a later writer overrides it
                    const pb2_tile_t& tl = w.tiles[(size_t)tile];
                    bool dup = false;
                    for (size_t k = 0; k < dst.size(); ++k) if (dst[k] == tl.src_ptr) dup = true;
                    if (!dup) { dst.push_back(tl.src_ptr); src.push_back(tl.dev_ptr); len.push_back(tl.bytes); }
                }
            }
        }
    }
    rc = pb2_engine_copy_batch(dev->engine, dst.data(), src.data(), len.data(), (int32_t)dst.size());   // stream-ordered after the bodies
    if (rc == PB2_SUCCESS) rc = pb2_engine_synchronize(dev->engine);
    if (rc != PB2_SUCCESS) ctx->last_error = std::string("submit lane: ") + pb2_engine_last_error(dev->engine);
    return rc;
}

// Host-resident tiles whose first use in the window is a READ, laid out contiguously on both sides, are moved by the
// copy engine in a few large cudaMemcpyAsync (parsec_cuda_memcpy_async, device_cuda_module.c:318-344, issues one per
// flow: 4096 calls of 256 KiB reach 29 GB/s on this box, one call per run 54 GB/s, worker CTAs 46 GB/s).
struct DmaRun { void* dev; size_t dpitch; const void* host; size_t hpitch; size_t width, rows; };

// plans the runs and marks their tiles resident; the copies are issued after the window's descriptors have been
// uploaded (small uploads queued behind a 256 MiB transfer on the same copy engine would block pb2_window_create)
static void dma_plan(pb2_device_module_t* dev, Window& w, std::vector<DmaRun>& runs) {
    const int64_t min_bytes = dev->ctx->mca["device_engine_dma_prefetch_min_bytes"];
    if (min_bytes <= 0) return;
    std::vector<int8_t> first((size_t)w.tiles.size(), -1);          // 1: first access reads the tile
    for (size_t i = 0; i < w.tasks.size(); ++i) {
        const pb2_task_t& t = w.tasks[i];
        for (int f = 0; f < t.nb_flows; ++f)
            if (t.tile[f] >= 0 && first[(size_t)t.tile[f]] < 0) first[(size_t)t.tile[f]] = (t.access[f] & PB2_FLOW_ACCESS_READ) ? 1 : 0;
    }
    std::vector<std::pair<uintptr_t, size_t>> cand;                  // (device address, tile index)
    for (size_t i = 0; i < w.tiles.size(); ++i) {
        const pb2_tile_t& tl = w.tiles[i];
        if (tl.state != PB2_TILE_INVALID || tl.src_kind != PB2_SRC_HOST || !tl.src_ptr || first[i] != 1) continue;
        pb2_data_copy_t* h = pb2i_host_copy(w.tile_data[i]);
        if (!h || !h->device_private) continue;
        cand.emplace_back((uintptr_t)tl.dev_ptr, i);
    }
    std::sort(cand.begin(), cand.end());
    auto host_of = [&](size_t c) { return (uintptr_t)pb2i_host_copy(w.tile_data[cand[c].second])->device_private; };
    size_t i = 0;
    while (i < cand.size()) {
        // longest run of equally sized tiles with constant strides on both sides, starting at candidate i
        const uint32_t width = w.tiles[cand[i].second].bytes;
        size_t j = i + 1;
        uintptr_t dpitch = width, hpitch = width;
        if (j < cand.size() && w.tiles[cand[j].second].bytes == width && host_of(j) > host_of(i)) {
            dpitch = cand[j].first - cand[i].first; hpitch = host_of(j) - host_of(i);
            if (dpitch >= width && hpitch >= width) {
                ++j;
                while (j < cand.size() && w.tiles[cand[j].second].bytes == width &&
                       cand[j].first - cand[j - 1].first == dpitch && host_of(j) - host_of(j - 1) == hpitch) ++j;
            } else { dpitch = hpitch = width; }
        }
        const size_t rows = j - i;
        if ((int64_t)((size_t)width * rows) >= min_bytes) {
            runs.push_back(DmaRun{reinterpret_cast<void*>(cand[i].first), dpitch, reinterpret_cast<const void*>(host_of(i)), hpitch, width, rows});
            for (size_t k = i; k < j; ++k) w.tiles[cand[k].second].state = PB2_TILE_VALID;   // resident when the window starts
        }
        i = j;
    }
}

// build one window from the pending tasks and start it (asynchronously)
static int launch_one(pb2_device_module_t* dev, bool* launched) {
    pb2_context_t* ctx = dev->ctx;
    *launched = false;
    InFlight* f = new InFlight();
    f->t_begin = now_ms();
    const size_t pipe = (size_t)std::max<int64_t>(1, ctx->mca["device_engine_pipeline"]);
    const size_t min_roots = (size_t)std::max<int64_t>(1, ctx->mca["device_engine_pipeline_min_roots"]);
    if (dev->pipe_chunk == 0 && pipe > 1 && dev->pending.size() >= min_roots)
        dev->pipe_chunk = (dev->pending.size() + pipe - 1) / pipe;
    const size_t max_roots = dev->pipe_chunk ? dev->pipe_chunk : (size_t)-1;
    int rc = build_window(dev, f->w, f->taken, max_roots);
    if (rc != PB2_SUCCESS || f->w.order.empty()) { delete f; return rc; }
    if (dev->pending.empty()) dev->pipe_chunk = 0;
    f->t_built = now_ms();
    if (!dev->dry_run && f->w.kind == 2) {
        rc = run_submit_lane(dev, f);
        if (rc != PB2_SUCCESS) { window_release(dev, f->w); delete f; return rc; }
    } else if (!dev->dry_run) {
        Window& w = f->w;
        const int32_t n = (int32_t)w.order.size();
        std::vector<DmaRun> runs;
        dma_plan(dev, w, runs);
        rc = pb2_window_create(dev->engine, &f->win, w.kind, w.tasks.data(), n, w.succ.data(), (int32_t)w.succ.size(),
                               w.tiles.data(), (int32_t)w.tiles.size(), w.ready.data(), (int32_t)w.ready.size());
        if (rc != PB2_SUCCESS) ctx->last_error = std::string("window_create: ") + pb2_engine_last_error(dev->engine);
        for (size_t r = 0; r < runs.size() && rc == PB2_SUCCESS; ++r) {
            rc = pb2_engine_prefetch_h2d(dev->engine, runs[r].dev, runs[r].dpitch, runs[r].host, runs[r].hpitch, runs[r].width, runs[r].rows);
            if (rc != PB2_SUCCESS) ctx->last_error = std::string("prefetch: ") + pb2_engine_last_error(dev->engine);
        }
        if (rc == PB2_SUCCESS && (rc = pb2_window_launch(f->win)) != PB2_SUCCESS)
            ctx->last_error = std::string("window launch: ") + pb2_engine_last_error(dev->engine);
        if (rc != PB2_SUCCESS) { if (f->win) pb2_window_destroy(f->win); window_release(dev, w); delete f; return rc; }
    }
    f->t_launched = now_ms();
    dev->inflight.push_back(f);
    *launched = true;
    return PB2_SUCCESS;
}

// wait for the oldest window and replay its bookkeeping
static int retire_one(pb2_device_module_t* dev) {
    pb2_context_t* ctx = dev->ctx;
    InFlight* f = reinterpret_cast<InFlight*>(dev->inflight.front());
    dev->inflight.pop_front();
    Window& w = f->w;
    const int32_t n = (int32_t)w.order.size();
    const double t_wait = now_ms();
    std::vector<int32_t> retire((size_t)n);
    std::vector<uint32_t> seen((size_t)n * PB2_MAX_FLOWS, 0);
    std::vector<uint64_t> result((size_t)n, 0);
    if (dev->dry_run || w.kind == 2) {
        // no device (dry run), or the submit lane, which ran its tasks in window order
        for (int32_t i = 0; i < n; ++i) retire[i] = i;
        if (!f->lane_seen.empty()) seen = f->lane_seen;
    } else {
        pb2_window_stats_t st{};
        int rc = pb2_window_wait(f->win, &st);
        if (rc == PB2_SUCCESS) rc = pb2_window_results(f->win, retire.data(), nullptr, nullptr, seen.data(), result.data(), nullptr, nullptr);
        if (rc == PB2_SUCCESS && dev->trace) {
            // window task i is the pool task w.order[i]
            std::vector<uint64_t> t0((size_t)n), t1((size_t)n);
            std::vector<uint32_t> sm((size_t)n);
            rc = pb2_window_trace(f->win, t0.data(), t1.data(), sm.data(), nullptr);
            if (rc == PB2_SUCCESS)
                for (int32_t i = 0; i < n; ++i) { pb2_htask_t* t = w.order[(size_t)i]; t->dev_t_start = t0[(size_t)i]; t->dev_t_end = t1[(size_t)i]; t->dev_smid = sm[(size_t)i]; }
            // the part records go to the pool of the task that led each entity, which they name by its pool task id
            int32_t nrec = 0;
            if (rc == PB2_SUCCESS) rc = pb2_window_part_trace(f->win, nullptr, 0, &nrec);
            std::vector<pb2_part_trace_t> rec((size_t)nrec);
            if (rc == PB2_SUCCESS && nrec) rc = pb2_window_part_trace(f->win, rec.data(), nrec, &nrec);
            if (rc == PB2_SUCCESS)
                for (pb2_part_trace_t r : rec) {
                    pb2_htask_t* t = w.order[(size_t)r.task];
                    r.task = t->id;
                    t->tp->part_trace.push_back(r);
                    t->tp->part_trace_device.push_back(dev->device_index);
                }
        }
        if (rc != PB2_SUCCESS) ctx->last_error = std::string("window run: ") + pb2_engine_last_error(dev->engine);
        pb2_window_destroy(f->win);
        if (rc != PB2_SUCCESS) { window_release(dev, w); delete f; return rc; }
        dev->st.kernel_ms_total += st.kernel_ms;
    }
    const double t_ran = now_ms();
    dev->st.windows_launched++;
    if (w.kind != 2) dev->st.tasks_released_on_device += (uint64_t)(n - (int32_t)w.ready.size());
    // the retire log is the order in which the host learns about completions
    for (int32_t i = 0; i < n; ++i) {
        pb2_htask_t* t = w.order[retire[i]];
        if (t->state != 2) { t->state = 2; t->selected_device = dev; t->load = time_estimate(t, dev); dev->st.device_load += t->load; }
        retire_task_bookkeeping(dev, w, t, &seen[(size_t)retire[i] * PB2_MAX_FLOWS], result[retire[i]]);
        pb2i_complete_execution(ctx, t, dev->device_index);      // __parsec_complete_execution, exactly once
    }
    // replicas go back on the LRUs: written ones are dirty (owned LRU) unless pushed out, read-only ones clean
    for (pb2_data_t* d : w.tile_data) {
        pb2_data_copy_t* g = d->device_copies[dev->device_index];
        if (!g) continue;
        // dirty = newer than the host copy.  (The reference decides by "a task wrote this flow and did not push it out",
        // device_gpu.c:3256-3289; the coherency state alone is not enough: a write to a replica that was already in
        // place leaves it SHARED, :1832-1836, and a SHARED replica on the clean list would be dropped without write-back.)
        const pb2_data_copy_t* h = pb2i_host_copy(d);
        const bool dirty = g->coherency_state == PB2_DATA_COHERENCY_OWNED || !h || g->version > h->version;
        pb2i_lru_push_back(dev, dirty ? 2 : 1, g);
    }
    window_release(dev, w);
    for (pb2_gpu_task_t* g : f->taken) { dev->mutex--; delete g; }    // release_device_task
    if (g_timing) fprintf(stderr, "pb2 window: %d tasks, build %.2f ms, create+launch %.2f ms, waited %.2f ms, retire %.2f ms\n",
                          n, f->t_built - f->t_begin, f->t_launched - f->t_built, t_ran - t_wait, now_ms() - t_ran);
    delete f;
    return PB2_SUCCESS;
}

// The manager's loop body (device_gpu.c:3438-3562), two windows deep: launch what is pending, then retire the oldest.
static int device_progress(pb2_device_module_t* dev) {
    const size_t depth = 2;
    bool launched = true;
    while (launched && !dev->pending.empty() && dev->inflight.size() < depth) {
        int rc = launch_one(dev, &launched);
        if (rc != PB2_SUCCESS) return rc;
    }
    if (!dev->inflight.empty()) return retire_one(dev);
    return PB2_SUCCESS;
}

extern "C" {

int pb2_taskpool_export_window(pb2_taskpool_t* tp, pb2_device_module_t* dev,
                               pb2_task_t* tasks, int32_t* ntasks, uint32_t* succ, int32_t* nsucc,
                               pb2_tile_t* tiles, int32_t* ntiles, int32_t* ready, int32_t* nready, int32_t* task_ids) {
    if (!tp || !dev || !ntasks || !nsucc || !ntiles || !nready) return PB2_ERR_BAD_PARAM;
    pb2_context_t* ctx = tp->ctx;
    if (!ctx->devices_frozen) pb2_mca_device_registration_complete(ctx);
    // hand every ready GPU task to the device like the worker loop would, but do not launch
    std::vector<pb2_htask_t*> keep;
    for (pb2_htask_t* t : ctx->ready) {
        if (t->tp != tp) { keep.push_back(t); continue; }
        const int d = pb2_select_best_device(ctx, t);
        if (d != dev->device_index) { keep.push_back(t); t->selected_device = nullptr; continue; }
        dev->st.device_load += t->load;
        pb2_gpu_task_t* g = new pb2_gpu_task_s();
        g->ec = t; g->pushout = t->pushout; g->nb_flows = (uint32_t)t->nb_flows;
        pb2_device_kernel_scheduler(dev, nullptr, g);
    }
    ctx->ready.swap(keep);
    Window w;
    std::vector<pb2_gpu_task_t*> taken;
    int rc = build_window(dev, w, taken, (size_t)-1);
    if (rc != PB2_SUCCESS) return rc;
    const bool fill = tasks && succ && tiles && ready &&
                      *ntasks >= (int32_t)w.tasks.size() && *nsucc >= (int32_t)w.succ.size() &&
                      *ntiles >= (int32_t)w.tiles.size() && *nready >= (int32_t)w.ready.size();
    if (fill) {
        memcpy(tasks, w.tasks.data(), w.tasks.size() * sizeof(pb2_task_t));
        memcpy(succ, w.succ.data(), w.succ.size() * sizeof(uint32_t));
        memcpy(tiles, w.tiles.data(), w.tiles.size() * sizeof(pb2_tile_t));
        memcpy(ready, w.ready.data(), w.ready.size() * sizeof(int32_t));
        if (task_ids) for (size_t i = 0; i < w.order.size(); ++i) task_ids[i] = w.order[i]->id;
    }
    *ntasks = (int32_t)w.tasks.size(); *nsucc = (int32_t)w.succ.size();
    *ntiles = (int32_t)w.tiles.size(); *nready = (int32_t)w.ready.size();
    // put everything back as it was: the tasks stay pending on the device, replicas go back to the clean LRU
    for (pb2_data_t* d : w.tile_data) {
        pb2_data_copy_t* g = d->device_copies[dev->device_index];
        if (g) pb2i_lru_push_back(dev, g->coherency_state == PB2_DATA_COHERENCY_OWNED ? 2 : 1, g);
    }
    window_release(dev, w);
    for (pb2_gpu_task_t* g : taken) dev->pending.push_back(g);
    return PB2_SUCCESS;
}

int pb2_device_memory_release(pb2_device_module_t* dev) {
    // parsec_device_flush_lru (device_gpu.c:1059-1077): write dirty replicas home, drop every replica
    if (!dev || !PB2_DEV_IS_GPU(dev->type)) return PB2_ERR_BAD_PARAM;
    while (w2r_flush(dev, 1 << 30) > 0) { }
    while (evict_one(dev)) { }
    dev->st.nb_evictions -= 0;
    return (dev->lru_count[1] + dev->lru_count[2]) == 0 ? PB2_SUCCESS : PB2_ERROR;
}

int pb2_device_data_advise(pb2_device_module_t* dev, pb2_data_t* data, int advice) {
    if (!dev || !data) return PB2_ERR_BAD_PARAM;
    switch (advice) {
    case PB2_DEV_DATA_ADVICE_PREFERRED_DEVICE:                      // device_gpu.c:760-763
        data->preferred_device = (int8_t)dev->device_index;
        return PB2_SUCCESS;
    case PB2_DEV_DATA_ADVICE_PREFETCH: {                            // device_gpu.c:722-758: bring a fresh replica in
        if (!PB2_DEV_IS_GPU(dev->type)) return PB2_ERR_NOT_SUPPORTED;
        pb2_data_copy_t* g = reserve_space(dev, data);
        if (!g) return PB2_ERR_OUT_OF_RESOURCE;
        pb2_data_copy_t* src = stage_in_source(dev, data);
        if (g->coherency_state != PB2_DATA_COHERENCY_INVALID && src && g->version >= src->version) return PB2_SUCCESS;
        if (!src || !src->device_private) return PB2_ERR_NOT_FOUND;
        int from = pb2_data_start_transfer_ownership_to_copy(dev->ctx, data, dev->device_index, PB2_FLOW_ACCESS_READ);
        g->readers--;                                               // a prefetch holds no reader
        if (from >= 0 && !dev->dry_run) {
            if (src->device_index == 0) pb2_engine_memcpy_h2d(dev->engine, g->device_private, src->device_private, data->span);
            else pb2_engine_memcpy_h2d(dev->engine, g->device_private, src->device_private, data->span);   // UVA: peer pointer works too
            pb2_engine_synchronize(dev->engine);
        }
        if (from >= 0) { dev->st.data_in_from_device[src->device_index] += data->span; g->version = src->version; }
        g->data_transfer_status = PB2_DATA_STATUS_COMPLETE_TRANSFER;
        pb2_data_end_transfer_ownership_to_copy(data, dev->device_index, PB2_FLOW_ACCESS_READ);
        pb2i_lru_push_back(dev, 1, g);
        return PB2_SUCCESS;
    }
    case PB2_DEV_DATA_ADVICE_WARMUP: {                              // NOT_IMPLEMENTED in the reference (:769-771); here: touch the LRU
        pb2_data_copy_t* g = data->device_copies[dev->device_index];
        if (!g || !g->lru_list) return PB2_ERR_NOT_FOUND;
        pb2i_lru_push_back(dev, g->lru_list, g);
        return PB2_SUCCESS;
    }
    default: return PB2_ERR_NOT_FOUND;
    }
}

int pb2_fini(pb2_context_t** pctx) {
    if (!pctx || !*pctx) return PB2_ERR_BAD_PARAM;
    pb2_context_t* ctx = *pctx;
    // windows still in flight (a wait that returned an error): let them finish on the device and drop them before the
    // tasks they point to go away
    for (auto* d : ctx->devices)
        while (!d->inflight.empty()) {
            InFlight* f = reinterpret_cast<InFlight*>(d->inflight.front());
            d->inflight.pop_front();
            if (f->win) pb2_window_destroy(f->win);
            window_release(d, f->w);
            for (pb2_gpu_task_t* g : f->taken) delete g;
            delete f;
        }
    while (!ctx->taskpools.empty()) pb2_taskpool_free(ctx->taskpools.back());
    if (ctx->mca["device_show_statistics"]) {                      // parsec_mca_device_fini, device.c:393-398
        std::vector<char> table((size_t)pb2_devices_statistics_string(ctx, nullptr, 0));
        pb2_devices_statistics_string(ctx, table.data(), table.size());
        fputs(table.data(), stdout);
    }
    for (auto* d : ctx->devices) {
        if (PB2_DEV_IS_GPU(d->type)) {
            for (int l = 1; l <= 2; ++l)
                while (d->lru_head[l]) { pb2_data_copy_t* c = d->lru_head[l]; pb2i_lru_remove(d, c); if (c->original) { c->original->device_copies[d->device_index] = nullptr; c->original->nb_copies--; } delete c; }
            if (d->engine) { if (d->slab) pb2_engine_free(d->engine, d->slab); pb2_engine_destroy(d->engine); }
        }
        delete d;
    }
    delete ctx;
    *pctx = nullptr;
    return PB2_SUCCESS;
}

}  // extern "C"
