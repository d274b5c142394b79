// pb2_device_module.cpp -- the GPU device module of the stand-alone runtime: device memory (reserve, evict, write
// back), then window building, launch and retire with the replay of the host-visible bookkeeping, i.e. the reference's
// push (reserve_space, device_gpu.c:1209, stage_in :1799) -> exec -> pop (:2943) -> epilog (:3179) for a whole window.
#include <algorithm>
#include <stdio.h>

#include "pb2_internal.hpp"
#include "pb2_engine_priv.hpp"

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
    if (!g) { g = pb2_data_copy_attach(d, dev->device_index); g->flags |= PB2_DATA_FLAG_PARSEC_OWNED; }
    g->device_private = slot;
    g->coherency_state = PB2_DATA_COHERENCY_INVALID; g->version = 0; g->readers = 0;
    g->data_transfer_status = PB2_DATA_STATUS_NOT_TRANSFER;
    return g;
}

// the highest version among the valid replicas of a datum (0 when none is valid).  The runtime makes replicas only on
// the host (index 0) and on its GPU modules, so the whole array reads the same as the context's devices.
static uint32_t newest_version(const pb2_data_t* d) {
    uint32_t newest = 0;
    for (const pb2_data_copy_t* c : d->device_copies)
        if (c && c->coherency_state != PB2_DATA_COHERENCY_INVALID && c->version > newest) newest = c->version;
    return newest;
}

// where would the bytes come from if this replica had to be filled now (stage_in source choice :1888-2008): a peer
// GPU replica of the newest version first, else the host copy
static pb2_data_copy_t* stage_in_source(pb2_device_module_t* dev, pb2_data_t* d, uint32_t newest) {
    for (size_t i = 2; i < dev->ctx->devices.size(); ++i) {
        pb2_data_copy_t* c = d->device_copies[i];
        if ((int)i == dev->device_index || !c || !c->device_private) continue;
        if (!(dev->peer_access_mask & (1u << i))) continue;
        if (c->coherency_state != PB2_DATA_COHERENCY_INVALID && c->version == newest &&
            c->data_transfer_status != PB2_DATA_STATUS_UNDER_TRANSFER) return c;
    }
    return pb2i_host_copy(d);
}

// What a window decided about one of its tiles, once, when it was built; indexed by the window tile id
struct TileUse {
    pb2_data_t* data;
    pb2_data_copy_t* src;                   // the copy stage-in reads; null when the replica is valid here or NEW
    bool first_reads;                       // the tile's first access in window order reads it
    bool staged;                            // the window moves it in for its first reader, whose replay clears it
};

// A window of the module, from taking its tasks to window_end; the module's inflight list holds the launched ones
struct pb2_device_window {
    int kind = 0;                           // 0 HBM kernel, 1 GEMM kernel, 2 the submit lane
    std::vector<pb2_gpu_task_t*> taken;     // the device tasks (kernel_scheduler's records) the window holds
    std::vector<pb2_htask_t*> order;        // window task i is the pool task order[i]
    std::vector<TileUse> use;
    std::vector<pb2_tile_t> tiles;
    std::vector<pb2_data_copy_t*> src_held; // peer replicas pinned (readers++) as stage-in sources until the window ends
    std::vector<pb2_task_t> tasks;
    std::vector<uint32_t> succ;
    std::vector<int32_t> ready;
    pb2_window_t* win = nullptr;            // the engine window, from create until it has been read back
    std::vector<uint32_t> lane_seen;        // kind 2: versions seen, filled when the lane ran
    double t_begin = 0, t_built = 0, t_launched = 0;
};

// The end of every window's life.  A window that ran puts its replicas back on the LRUs first -- written ones are
// dirty (owned LRU) unless pushed out, read-only ones clean -- and gives its device tasks back (release_device_task).
// Every other path leaves the replicas where they are and drops the device tasks without re-queuing them.
static void window_end(pb2_device_module_t* dev, pb2_device_window* w, bool ran) {
    if (w->win) pb2_window_destroy(w->win);
    for (const TileUse& u : w->use) {
        pb2_data_copy_t* g = u.data->device_copies[dev->device_index];
        if (!g) continue;
        if (ran) {
            // dirty = newer than the host copy.  (The reference decides by "a task wrote this flow and did not push it
            // out", device_gpu.c:3256-3289; the coherency state alone is not enough: a write to a replica that was
            // already in place leaves it SHARED, :1832-1836, and a SHARED replica on the clean list would be dropped
            // without write-back.)
            const pb2_data_copy_t* h = pb2i_host_copy(u.data);
            const bool dirty = g->coherency_state == PB2_DATA_COHERENCY_OWNED || !h || g->version > h->version;
            pb2i_lru_push_back(dev, dirty ? 2 : 1, g);
        }
        g->window_tile = -1; g->window_owner = nullptr;
    }
    for (pb2_data_copy_t* c : w->src_held) c->readers--;
    for (pb2_htask_t* t : w->order) t->window_index = -1;
    for (pb2_gpu_task_t* g : w->taken) { if (ran) dev->mutex--; delete g; }
    delete w;
}

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

// Take the dependency-closed window reachable from the pending tasks of one taskpool, reserving a slot for every tile
// it touches.  An engine window takes tile GEMMs and HBM bodies together, so that a GEMM chain and the element-wise
// tasks around it are released on the device instead of through the host; its kind is decided by the closure: 1 (the
// GEMM kernel, which also runs HBM bodies) when it holds a GEMM task -- a bf16 tile GEMM, or a task of a GEMM-worker
// body (PB2_LINK_GEMM_BODIES), which runs in GEMM windows only -- else 0.  User submit tasks never mix with engine
// tasks.  Unless the module linked its bodies with PB2_LINK_GEMM_WINDOWS, tasks of linked bodies (which then run in the
// linked HBM kernel only) never mix with GEMM tasks: the first of the two kinds the closure takes in keeps the other out
// of this window.
static int take_closure(pb2_device_module_t* dev, pb2_device_window& w, size_t max_roots) {
    if (dev->pending.empty()) return PB2_SUCCESS;
    pb2_taskpool_t* const tp = dev->pending.front()->ec->tp;
    const bool want_user = dev->pending.front()->ec->body == PB2_BODY_USER;      // the host-driven stream lane
    int engine_side = 0;                        // PB2_BODY_GEMM_BF16 or PB2_BODY_LINKED_0 once the window holds one
    auto fits = [&](const pb2_htask_t* t) {
        if ((t->body == PB2_BODY_USER) != want_user) return false;
        const int side = dev->linked_gemm ? 0 : t->body == PB2_BODY_GEMM_BF16 ? PB2_BODY_GEMM_BF16
                                              : pb2::is_linked_body(t->body) ? PB2_BODY_LINKED_0 : 0;
        if (side && engine_side && side != engine_side) return false;
        if (side) engine_side = side;
        return true;
    };
    bool has_gemm = false;
    std::deque<pb2_htask_t*> queue;
    std::deque<pb2_gpu_task_t*> keep;
    for (pb2_gpu_task_t* g : dev->pending) {
        if (w.taken.size() < max_roots && g->ec->tp == tp && fits(g->ec)) { queue.push_back(g->ec); w.taken.push_back(g); }
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
                    // tasks join in window order, so this flow is the tile's first access in the window
                    g->window_tile = (int32_t)w.use.size();
                    g->window_owner = &w;
                    w.use.push_back(TileUse{d, nullptr, (t->access[f] & PB2_FLOW_ACCESS_READ) != 0, false});
                    fresh.push_back(g);
                }
            }
        }
        if (!ok) {
            // no room: this task (and everything behind it) waits for the next window (HOOK_RETURN_AGAIN)
            full = true;
            for (pb2_data_copy_t* g : fresh) {
                g->window_tile = -1; g->window_owner = nullptr; w.use.pop_back();
                // a slot reserve_space has just allocated for this task is on no list yet: put it where eviction finds it
                if (g->lru_list == 0) pb2i_lru_push_back(dev, (g->coherency_state == PB2_DATA_COHERENCY_OWNED && g->version > 0) ? 2 : 1, g);
            }
            continue;
        }
        t->window_index = (int32_t)w.order.size();
        w.order.push_back(t);
        has_gemm |= t->body == PB2_BODY_GEMM_BF16 ||
                    (pb2::is_linked_body(t->body) && ((dev->linked_gemm_bodies >> (t->body - PB2_BODY_LINKED_0)) & 1u));
        for (uint32_t s : t->succ) {
            pb2_htask_t* n = &tp->tasks[PB2_SUCC_TASK(s)];
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
        for (pb2_gpu_task_t* g : w.taken) { if (g->ec->window_index >= 0) in.push_back(g); else dev->pending.push_back(g); }
        w.taken.swap(in);
    }
    if (w.order.empty() && dev->inflight.empty()) {                 // else everything waits for the window that is running
        dev->ctx->last_error = "device memory too small for a single task"; return PB2_ERR_OUT_OF_RESOURCE;
    }
    return PB2_SUCCESS;
}

// Decide each tile's state, version and stage-in source by VERSION, and take its replica off the LRUs until the
// window ends
static int describe_tiles(pb2_device_module_t* dev, pb2_device_window& w) {
    w.tiles.resize(w.use.size());
    for (size_t i = 0; i < w.use.size(); ++i) {
        TileUse& u = w.use[i];
        pb2_data_t* d = u.data;
        pb2_data_copy_t* g = d->device_copies[dev->device_index];
        pb2i_lru_remove(dev, g);                                    // in use: off the lists until retire
        pb2_tile_t& tl = w.tiles[i];
        memset(&tl, 0, sizeof tl);
        tl.dev_ptr = g->device_private;
        if (d->span > 0xffffffffull) { dev->ctx->last_error = "tile larger than 4 GiB (pb2_tile_t::bytes is 32-bit)"; return PB2_ERR_VALUE_OUT_OF_BOUNDS; }
        tl.bytes = (uint32_t)d->span;
        const uint32_t newest = newest_version(d);
        const bool valid_here = g->coherency_state != PB2_DATA_COHERENCY_INVALID && g->version >= newest;
        pb2_data_copy_t* src = valid_here ? nullptr : stage_in_source(dev, d, newest);
        // a peer GPU's replica that this window will read from must stay where it is until the window has retired: hold
        // a reader on it, like the reference does for D2D sources (device_gpu.c:1925-1975, released :2461-2526)
        if (src && src->device_index >= 2 && src->device_index != dev->device_index) { src->readers++; w.src_held.push_back(src); }
        pb2_data_copy_t* h = pb2i_host_copy(d);
        const bool is_new = (d->dc == nullptr) && h && h->version == 0 && newest == 0;   // NEW: nothing to pull (:2049)
        if (valid_here) { tl.state = PB2_TILE_VALID; tl.version = g->version; }
        else if (is_new) { tl.state = PB2_TILE_VALID; tl.version = 0; }
        else { tl.state = PB2_TILE_INVALID; tl.version = src ? src->version : 0; }
        u.src = is_new ? nullptr : src;
        u.staged = tl.state == PB2_TILE_INVALID && src != nullptr;
        tl.src_kind = (src && src->device_index >= 2) ? PB2_SRC_PEER : PB2_SRC_HOST;
        // the home of the tile for pushout is always the host copy; a peer source is only used for stage-in
        void* host_alias = dev->dry_run ? (h ? h->device_private : nullptr) : pb2i_device_visible_host_ptr(dev, d);
        tl.src_ptr = (tl.src_kind == PB2_SRC_PEER) ? src->device_private : host_alias;
    }
    return PB2_SUCCESS;
}

// The window's task descriptors and the CSR of its in-window edges
static void encode_tasks(pb2_device_module_t* dev, pb2_device_window& w) {
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
            pb2_htask_t* n = &t->tp->tasks[PB2_SUCC_TASK(s)];
            if (n->window_index >= 0) w.succ.push_back(PB2_SUCC_MAKE(n->window_index, PB2_SUCC_FLOW(s)));
        }
        o.succ_count = (int32_t)w.succ.size() - o.succ_begin;
        if (t->state == 2) w.ready.push_back((int32_t)i);          // handed over by kernel_scheduler: ready now
    }
}

static int build_window(pb2_device_module_t* dev, pb2_device_window& w, size_t max_roots) {
    int rc = take_closure(dev, w, max_roots);
    if (rc != PB2_SUCCESS || w.order.empty()) return rc;
    if ((rc = describe_tiles(dev, w)) != PB2_SUCCESS) return rc;
    encode_tasks(dev, w);
    return PB2_SUCCESS;
}

// Host-visible bookkeeping of one retired task, replayed in retire order exactly as the reference's manager
// thread would have done it around the task: stage_in (device_gpu.c:1799-2165) + callback_complete_push
// (:2358-2573) for every flow, then kernel_pop (:2943-3173) + kernel_epilog (:3179-3292).
static void retire_task_bookkeeping(pb2_device_module_t* dev, pb2_device_window& w, pb2_htask_t* t, const uint32_t* seen, uint64_t result) {
    pb2_context_t* ctx = dev->ctx;
    const int di = dev->device_index;
    for (int f = 0; f < t->nb_flows; ++f) {
        pb2_data_t* d = t->data[f];
        t->seen_version[f] = seen[f];
        if (!d) continue;
        pb2_data_copy_t* g = d->device_copies[di];
        TileUse& u = w.use[(size_t)g->window_tile];
        const uint8_t acc = t->access[f];
        pb2_data_copy_t* in = t->data_in[f] ? t->data_in[f] : pb2i_host_copy(d);
        // the copy the task was given as input may have been evicted (and written back) since: the bytes then came from
        // the source chosen when the window was built (stage_in_source: newest valid replica, normally the host copy)
        if (in->coherency_state == PB2_DATA_COHERENCY_INVALID && in->device_index >= 2) in = u.src ? u.src : pb2i_host_copy(d);
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
            pb2_data_copy_t* cand = (!(acc & PB2_FLOW_ACCESS_WRITE) && u.src) ? u.src : in;
            int from = pb2_data_start_transfer_ownership_to_copy(ctx, d, (uint8_t)di, acc);
            if (d->dc == nullptr && in->device_index == 0 && in->version == 0) from = -1;   // NEW, untouched (:2049-2052)
            // The window decided by VERSION whether this replica had to be refreshed (describe_tiles: valid_here) and
            // the kernel moved the bytes for the first reader.  The coherency states alone can say "no transfer": a
            // write to a replica that is already in place leaves the other GPUs' older replicas SHARED (:1832-1836).
            // The replay follows what was done.
            if ((acc & PB2_FLOW_ACCESS_READ) && u.staged) {
                u.staged = false;
                if (u.src) cand = u.src;
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

// Tasks whose CUDA chore is a user `submit` function (PB2_BODY_USER): the host does for them what the reference's
// manager does for every task -- stage the inputs in (kernel_push), call submit on the stream (kernel_exec,
// device_gpu.c:2873-2934), write pushout flows back (kernel_pop) -- but for a whole dependency-closed chain of
// them at once and with batched copies: one copy kernel for all stage-ins, one for all write-backs.
static int run_submit_lane(pb2_device_module_t* dev, pb2_device_window& w) {
    pb2_context_t* ctx = dev->ctx;
    const size_t n = w.order.size();
    std::vector<void*> dst; std::vector<const void*> src; std::vector<uint64_t> len;
    for (size_t i = 0; i < w.tiles.size(); ++i) {
        const pb2_tile_t& tl = w.tiles[i];
        if (tl.state != PB2_TILE_INVALID || !w.use[i].first_reads || !tl.src_ptr) continue;
        dst.push_back(tl.dev_ptr); src.push_back(tl.src_ptr); len.push_back(tl.bytes);
    }
    int rc = pb2_engine_copy_batch(dev->engine, dst.data(), src.data(), len.data(), (int32_t)dst.size());
    if (rc != PB2_SUCCESS) { ctx->last_error = std::string("submit lane stage-in: ") + pb2_engine_last_error(dev->engine); return rc; }
    void* stream = pb2_engine_get_stream(dev->engine);
    std::vector<uint32_t> ver(w.tiles.size());
    for (size_t i = 0; i < w.tiles.size(); ++i) ver[i] = w.tiles[i].version;
    w.lane_seen.assign(n * PB2_MAX_FLOWS, 0);
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
            w.lane_seen[i * PB2_MAX_FLOWS + (size_t)fl] = ver[(size_t)tile];
            if (w.tasks[i].access[fl] & PB2_FLOW_ACCESS_WRITE) {
                ver[(size_t)tile]++;
                if (w.tasks[i].access[fl] & PB2_FLOW_PUSHOUT) {        // newest version goes home; a later writer overrides it
                    const pb2_tile_t& tl = w.tiles[(size_t)tile];
                    if (std::find(dst.begin(), dst.end(), tl.src_ptr) == dst.end()) { dst.push_back(tl.src_ptr); src.push_back(tl.dev_ptr); len.push_back(tl.bytes); }
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
static void dma_plan(pb2_device_module_t* dev, pb2_device_window& w, std::vector<DmaRun>& runs) {
    const int64_t min_bytes = dev->ctx->mca["device_engine_dma_prefetch_min_bytes"];
    if (min_bytes <= 0) return;
    std::vector<std::pair<uintptr_t, size_t>> cand;                  // (device address, tile index)
    for (size_t i = 0; i < w.tiles.size(); ++i) {
        const pb2_tile_t& tl = w.tiles[i];
        if (tl.state != PB2_TILE_INVALID || tl.src_kind != PB2_SRC_HOST || !tl.src_ptr || !w.use[i].first_reads) continue;
        pb2_data_copy_t* h = pb2i_host_copy(w.use[i].data);
        if (!h || !h->device_private) continue;
        cand.emplace_back((uintptr_t)tl.dev_ptr, i);
    }
    std::sort(cand.begin(), cand.end());
    auto host_of = [&](size_t c) { return (uintptr_t)pb2i_host_copy(w.use[cand[c].second].data)->device_private; };
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
    pb2_device_window* w = new pb2_device_window();
    w->t_begin = pb2i_now_ms();
    const size_t pipe = (size_t)std::max<int64_t>(1, ctx->mca["device_engine_pipeline"]);
    const size_t min_roots = (size_t)std::max<int64_t>(1, ctx->mca["device_engine_pipeline_min_roots"]);
    if (dev->pipe_chunk == 0 && pipe > 1 && dev->pending.size() >= min_roots)
        dev->pipe_chunk = (dev->pending.size() + pipe - 1) / pipe;
    const size_t max_roots = dev->pipe_chunk ? dev->pipe_chunk : (size_t)-1;
    int rc = build_window(dev, *w, max_roots);
    if (rc != PB2_SUCCESS || w->order.empty()) { window_end(dev, w, false); return rc; }
    if (dev->pending.empty()) dev->pipe_chunk = 0;
    w->t_built = pb2i_now_ms();
    if (!dev->dry_run && w->kind == 2) {
        rc = run_submit_lane(dev, *w);
    } else if (!dev->dry_run) {
        std::vector<DmaRun> runs;
        dma_plan(dev, *w, runs);
        rc = pb2_window_create(dev->engine, &w->win, w->kind, w->tasks.data(), (int32_t)w->order.size(), w->succ.data(), (int32_t)w->succ.size(),
                               w->tiles.data(), (int32_t)w->tiles.size(), w->ready.data(), (int32_t)w->ready.size());
        if (rc != PB2_SUCCESS) ctx->last_error = std::string("window_create: ") + pb2_engine_last_error(dev->engine);
        for (size_t r = 0; r < runs.size() && rc == PB2_SUCCESS; ++r) {
            rc = pb2_engine_prefetch_h2d(dev->engine, runs[r].dev, runs[r].dpitch, runs[r].host, runs[r].hpitch, runs[r].width, runs[r].rows);
            if (rc != PB2_SUCCESS) ctx->last_error = std::string("prefetch: ") + pb2_engine_last_error(dev->engine);
        }
        if (rc == PB2_SUCCESS && (rc = pb2_window_launch(w->win)) != PB2_SUCCESS)
            ctx->last_error = std::string("window launch: ") + pb2_engine_last_error(dev->engine);
    }
    if (rc != PB2_SUCCESS) { window_end(dev, w, false); return rc; }
    w->t_launched = pb2i_now_ms();
    dev->inflight.push_back(w);
    *launched = true;
    return PB2_SUCCESS;
}

// device_engine_trace: the time stamps of window task i go to the pool task w.order[i], and the part records to the
// pool of the task that led each entity, which they name by its pool task id
static int read_window_trace(pb2_device_module_t* dev, pb2_device_window& w) {
    const size_t n = w.order.size();
    std::vector<uint64_t> t0(n), t1(n);
    std::vector<uint32_t> sm(n);
    int rc = pb2_window_trace(w.win, t0.data(), t1.data(), sm.data(), nullptr);
    if (rc != PB2_SUCCESS) return rc;
    for (size_t i = 0; i < n; ++i) { pb2_htask_t* t = w.order[i]; t->dev_t_start = t0[i]; t->dev_t_end = t1[i]; t->dev_smid = sm[i]; }
    int32_t nrec = 0;
    if ((rc = pb2_window_part_trace(w.win, nullptr, 0, &nrec)) != PB2_SUCCESS) return rc;
    std::vector<pb2_part_trace_t> rec((size_t)nrec);
    if (nrec && (rc = pb2_window_part_trace(w.win, rec.data(), nrec, &nrec)) != PB2_SUCCESS) return rc;
    for (pb2_part_trace_t r : rec) {
        pb2_htask_t* t = w.order[(size_t)r.task];
        r.task = t->id;
        t->tp->part_trace.push_back(r);
        t->tp->part_trace_device.push_back(dev->device_index);
    }
    return PB2_SUCCESS;
}

// wait for the oldest window and replay its bookkeeping
static int retire_one(pb2_device_module_t* dev) {
    pb2_context_t* ctx = dev->ctx;
    pb2_device_window* w = dev->inflight.front();
    dev->inflight.pop_front();
    const int32_t n = (int32_t)w->order.size();
    const double t_wait = pb2i_now_ms();
    std::vector<int32_t> retire((size_t)n);
    std::vector<uint32_t> seen((size_t)n * PB2_MAX_FLOWS, 0);
    std::vector<uint64_t> result((size_t)n, 0);
    if (dev->dry_run || w->kind == 2) {
        // no device (dry run), or the submit lane, which ran its tasks in window order
        for (int32_t i = 0; i < n; ++i) retire[i] = i;
        if (!w->lane_seen.empty()) seen = w->lane_seen;
    } else {
        pb2_window_stats_t st{};
        int rc = pb2_window_wait(w->win, &st);
        if (rc == PB2_SUCCESS) rc = pb2_window_results(w->win, retire.data(), nullptr, nullptr, seen.data(), result.data(), nullptr, nullptr);
        if (rc == PB2_SUCCESS && dev->trace) rc = read_window_trace(dev, *w);
        if (rc != PB2_SUCCESS) ctx->last_error = std::string("window run: ") + pb2_engine_last_error(dev->engine);
        pb2_window_destroy(w->win); w->win = nullptr;
        if (rc != PB2_SUCCESS) { window_end(dev, w, false); return rc; }
        dev->st.kernel_ms_total += st.kernel_ms;
    }
    const double t_ran = pb2i_now_ms();
    dev->st.windows_launched++;
    if (w->kind != 2) dev->st.tasks_released_on_device += (uint64_t)(n - (int32_t)w->ready.size());
    // the retire log is the order in which the host learns about completions
    for (int32_t i = 0; i < n; ++i) {
        pb2_htask_t* t = w->order[retire[i]];
        if (t->state != 2) { t->state = 2; t->selected_device = dev; t->load = pb2i_time_estimate(t, dev); dev->st.device_load += t->load; }
        retire_task_bookkeeping(dev, *w, t, &seen[(size_t)retire[i] * PB2_MAX_FLOWS], result[retire[i]]);
        pb2i_complete_execution(ctx, t, dev->device_index);      // __parsec_complete_execution, exactly once
    }
    const double build_ms = w->t_built - w->t_begin, launch_ms = w->t_launched - w->t_built;
    window_end(dev, w, true);
    if (pb2i_timing) fprintf(stderr, "pb2 window: %d tasks, build %.2f ms, create+launch %.2f ms, waited %.2f ms, retire %.2f ms\n",
                             n, build_ms, launch_ms, t_ran - t_wait, pb2i_now_ms() - t_ran);
    return PB2_SUCCESS;
}

// The manager's loop body (device_gpu.c:3438-3562), two windows deep: launch what is pending, then retire the oldest.
int pb2i_device_progress(pb2_device_module_t* dev) {
    const size_t depth = 2;
    bool launched = true;
    while (launched && !dev->pending.empty() && dev->inflight.size() < depth) {
        int rc = launch_one(dev, &launched);
        if (rc != PB2_SUCCESS) return rc;
    }
    if (!dev->inflight.empty()) return retire_one(dev);
    return PB2_SUCCESS;
}

// windows still in flight (a wait that returned an error): let them finish on the device and drop them before the
// tasks they point to go away
void pb2i_device_drain(pb2_device_module_t* dev) {
    for (pb2_device_window* w : dev->inflight) window_end(dev, w, false);
    dev->inflight.clear();
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
    pb2_device_window* w = new pb2_device_window();
    int rc = build_window(dev, *w, (size_t)-1);
    if (rc != PB2_SUCCESS) { window_end(dev, w, false); return rc; }
    const bool fill = tasks && succ && tiles && ready &&
                      *ntasks >= (int32_t)w->tasks.size() && *nsucc >= (int32_t)w->succ.size() &&
                      *ntiles >= (int32_t)w->tiles.size() && *nready >= (int32_t)w->ready.size();
    if (fill) {
        memcpy(tasks, w->tasks.data(), w->tasks.size() * sizeof(pb2_task_t));
        memcpy(succ, w->succ.data(), w->succ.size() * sizeof(uint32_t));
        memcpy(tiles, w->tiles.data(), w->tiles.size() * sizeof(pb2_tile_t));
        memcpy(ready, w->ready.data(), w->ready.size() * sizeof(int32_t));
        if (task_ids) for (size_t i = 0; i < w->order.size(); ++i) task_ids[i] = w->order[i]->id;
    }
    *ntasks = (int32_t)w->tasks.size(); *nsucc = (int32_t)w->succ.size();
    *ntiles = (int32_t)w->tiles.size(); *nready = (int32_t)w->ready.size();
    // put everything back as it was: the tasks stay pending on the device, replicas go back to the clean LRU
    for (const TileUse& u : w->use) {
        pb2_data_copy_t* g = u.data->device_copies[dev->device_index];
        if (g) pb2i_lru_push_back(dev, g->coherency_state == PB2_DATA_COHERENCY_OWNED ? 2 : 1, g);
    }
    for (pb2_gpu_task_t* g : w->taken) dev->pending.push_back(g);
    w->taken.clear();
    window_end(dev, w, false);
    return PB2_SUCCESS;
}

int pb2_device_memory_release(pb2_device_module_t* dev) {
    // parsec_device_flush_lru (device_gpu.c:1059-1077): write dirty replicas home, drop every replica
    if (!dev || !PB2_DEV_IS_GPU(dev->type)) return PB2_ERR_BAD_PARAM;
    while (w2r_flush(dev, 1 << 30) > 0) { }
    while (evict_one(dev)) { }
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
        pb2_data_copy_t* src = stage_in_source(dev, data, newest_version(data));
        if (g->coherency_state != PB2_DATA_COHERENCY_INVALID && src && g->version >= src->version) return PB2_SUCCESS;
        if (!src || !src->device_private) return PB2_ERR_NOT_FOUND;
        int from = pb2_data_start_transfer_ownership_to_copy(dev->ctx, data, dev->device_index, PB2_FLOW_ACCESS_READ);
        g->readers--;                                               // a prefetch holds no reader
        if (from >= 0 && !dev->dry_run) {
            pb2_engine_memcpy_h2d(dev->engine, g->device_private, src->device_private, data->span);   // UVA: a peer pointer works too
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

}  // extern "C"
