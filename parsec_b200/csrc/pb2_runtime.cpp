// pb2_runtime.cpp -- host side of the engine: data coherency, device heap + LRUs, the context and its MCA
// parameters, the device registry and selection, scheduling, CPU execution, task completion and dependency release.
// It mirrors the reference's control flow around the device boundary
//   worker:  __parsec_execute (scheduling.c:126-206) -> chore hook -> dev->kernel_scheduler (device_gpu.c:3375)
//   device:  push -> exec -> pop -> epilog, in the GPU device module (pb2_device_module.cpp)
//   worker:  __parsec_complete_execution (scheduling.c:469-505) -> release_deps (parsec.c:1836)
// but hands whole dependency-closed sets of GPU tasks ("windows") to the persistent kernel, so the per-task and
// per-edge host round trips of the reference only remain at window boundaries and for CPU incarnations.
#include <algorithm>
#include <stdio.h>

#include "pb2_internal.hpp"
#include "pb2_engine_priv.hpp"

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
    return pb2_device_link_bodies_checked(dev, image, bytes, format, sliceable, 0);
}
int pb2_device_link_bodies_checked(pb2_device_module_t* dev, const void* image, size_t bytes, int format, uint32_t sliceable,
                                   uint32_t checked) {
    return pb2_device_link_bodies_ex(dev, image, bytes, format, sliceable, checked, 0);
}
int pb2_device_link_bodies_ex(pb2_device_module_t* dev, const void* image, size_t bytes, int format, uint32_t sliceable,
                              uint32_t checked, uint32_t flags) {
    if (!dev || !PB2_DEV_IS_GPU(dev->type)) return PB2_ERR_BAD_PARAM;
    pb2_context_t* ctx = dev->ctx;
    if (const char* why = link_args_error(image, bytes, format, sliceable, checked, flags)) { ctx->last_error = why; return PB2_ERR_BAD_PARAM; }
    if (dev->linked) { ctx->last_error = "the module has linked an image already (one per module)"; return PB2_ERR_EXISTS; }
    if (dev->st.windows_launched) { ctx->last_error = "linked bodies must be linked before the module's first window"; return PB2_ERR_NOT_SUPPORTED; }
    if (!dev->dry_run) {
        const int rc = pb2_engine_link_bodies_ex(dev->engine, image, bytes, format, sliceable, checked, flags);
        if (rc != PB2_SUCCESS) { ctx->last_error = pb2_engine_last_error(dev->engine); return rc; }
    }
    dev->linked = true;
    dev->linked_gemm = (flags & PB2_LINK_GEMM_WINDOWS) != 0;
    dev->linked_readers = link_readers(flags);
    dev->linked_gemm_bodies = link_gemm_bodies(flags);
    dev->linked_gemm_body_entry = (flags & PB2_LINK_GEMM_BODY_ENTRY) != 0;
    return PB2_SUCCESS;
}

// The module's windows are planned by its engine, which holds the counts; the module keeps them too, so that a dry-run
// module records them.
int pb2_device_set_gemm_body_parts(pb2_device_module_t* dev, int body, int32_t nparts) {
    if (!dev || !PB2_DEV_IS_GPU(dev->type)) return PB2_ERR_BAD_PARAM;
    int rc;
    if (const char* why = gemm_body_parts_error(dev->linked, dev->linked_gemm_bodies, body, nparts, &rc)) {
        dev->ctx->last_error = why;
        return rc;
    }
    if (!dev->dry_run && (rc = pb2_engine_set_gemm_body_parts(dev->engine, body, nparts)) != PB2_SUCCESS) {
        dev->ctx->last_error = pb2_engine_last_error(dev->engine);
        return rc;
    }
    dev->gemm_body_parts[body - PB2_BODY_LINKED_0] = nparts;
    return PB2_SUCCESS;
}
int pb2_device_gemm_body_parts(pb2_device_module_t* dev, int body) {
    if (!dev || !PB2_DEV_IS_GPU(dev->type) || body < PB2_BODY_LINKED_0 || body > PB2_BODY_LINKED_7) return PB2_ERR_BAD_PARAM;
    return dev->gemm_body_parts[body - PB2_BODY_LINKED_0];
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
int64_t pb2i_time_estimate(pb2_htask_t* t, pb2_device_module_t* d) { (void)t; return d->st.time_estimate_default; }

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
            best_eta = (int64_t)((float)(rdata_dev->st.device_load + pb2i_time_estimate(t, rdata_dev)) * skew);
        }
        for (int d = (int)ctx->devices.size() - 1; d >= 0; d--) {
            pb2_device_module_t* dev = usable(d);
            if (!dev || (dev->type & PB2_DEV_RECURSIVE)) continue;
            const int64_t eta = dev->st.device_load + pb2i_time_estimate(t, dev);
            if (best_eta > eta) {
                if (best_index != -1 && !PB2_DEV_IS_GPU(dev->type) && !ctx->mca["device_load_balance_allow_cpu"]) continue;
                best_index = d; best_eta = eta;
            }
        }
        if (best_index < 0) return -1;
        t->selected_device = ctx->devices[best_index];
    }
selected:
    t->load = pb2i_time_estimate(t, t->selected_device);
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
        const double t_sched = pb2i_now_ms();
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
        if (pb2i_timing && nready0) fprintf(stderr, "pb2 wait: dispatched %zu ready tasks in %.2f ms\n", nready0, pb2i_now_ms() - t_sched);
        for (auto* d : ctx->devices) {
            if (!PB2_DEV_IS_GPU(d->type) || (d->pending.empty() && d->inflight.empty())) continue;
            int rc = pb2i_device_progress(d);
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

int pb2_fini(pb2_context_t** pctx) {
    if (!pctx || !*pctx) return PB2_ERR_BAD_PARAM;
    pb2_context_t* ctx = *pctx;
    for (auto* d : ctx->devices) pb2i_device_drain(d);
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
