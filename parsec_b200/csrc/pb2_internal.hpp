// pb2_internal.hpp -- private structures of the host side (pb2_runtime.cpp, pb2_device_module.cpp, pb2_dsl.cpp).
#pragma once
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <chrono>
#include <deque>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/pb2_parsec.h"

// ---------------------------------------------------------------------------------------------
// Device heap: the segment allocator of parsec/utils/zone_malloc.c restated (unit-granular, smallest
// sufficient free segment first, most recently freed first among equals, coalescing free).
// ---------------------------------------------------------------------------------------------
struct pb2_zone {
    struct Seg { int status; int nb_units; int nb_prev; uint64_t stamp; };
    enum { UNDEF = 0, EMPTY = 1, FULL = 2 };
    char* base = nullptr;
    size_t unit_size = 0;
    int max_segment = 0;
    uint64_t clock = 1;
    std::vector<Seg> seg;
    // free segments ordered by (nb_units asc, stamp desc): begin() of lower_bound is the reference's choice
    struct Key { int nb_units; uint64_t inv_stamp; bool operator<(const Key& o) const { return nb_units != o.nb_units ? nb_units < o.nb_units : inv_stamp < o.inv_stamp; } };
    std::map<Key, int> free_by_size;

    void init(void* base_ptr, int max_seg, size_t unit);
    void* malloc(size_t size);
    int free(void* ptr);
    size_t in_use() const;
private:
    void add_free(int tid);
    void del_free(int tid);
};

struct pb2_data_collection_s {
    pb2_context_t* ctx = nullptr;
    int elt_bytes = 1;
    // parsec_matrix_block_cyclic_t / parsec_tiled_matrix_t / grid_2Dcyclic_t fields (same names)
    int myrank = 0, mb = 1, nb = 1, lm = 1, ln = 1, i = 0, j = 0, m = 1, n = 1;
    int P = 1, Q = 1, kp = 1, kq = 1, ip = 0, jq = 0;
    int lmt = 0, lnt = 0, mt = 0, nt = 0, rrank = 0, crank = 0;
    int nb_elem_r = 0, nb_elem_c = 0, nb_local_tiles = 0, llm = 0, lln = 0;
    int64_t bsiz = 0;
    void* mat = nullptr;
    std::vector<pb2_data_t*> data_map;        // [nb_local_tiles], created on demand
    uint32_t memory_registration_status = 0;  // one bit per device, device_cuda_module.c:183-238
    std::map<int, void*> device_alias;        // device index -> device-visible alias of mat
};

struct pb2_task_class_s {
    std::string name;
    int task_class_id = 0;
    int nb_flows = 0;
    int32_t flow_ops[PB2_MAX_FLOWS] = {0, 0, 0, 0};   // DTD: PB2_INPUT/... | PB2_AFFINITY
    uint8_t chore_types = 0;                          // PB2_DEV_* with an incarnation
    int gpu_body = -1;
    pb2_cpu_hook_t cpu_hook = nullptr;
    pb2_gpu_submit_t submit = nullptr;                // PB2_BODY_USER: the user's own stream-enqueue function
    bool use_mask = false;
};

// Successor list of a host task: up to 8 out-edges inline (a broadcast of Ex05 has 8, a GEMM chain member 1-3), heap
// beyond that.  The reference keeps out-edges implicit in generated code; the per-task malloc of a std::vector was
// the largest single cost of building a PTG pool.
struct pb2_succ_list {
    uint32_t inl[8];
    uint32_t* heap = nullptr;
    uint32_t n = 0, cap = 8;
    pb2_succ_list() = default;
    pb2_succ_list(const pb2_succ_list&) = delete;
    pb2_succ_list& operator=(const pb2_succ_list&) = delete;
    ~pb2_succ_list() { free(heap); }
    void push_back(uint32_t v) {
        if (n == cap) {
            const uint32_t ncap = cap * 2;
            uint32_t* nh = static_cast<uint32_t*>(malloc(sizeof(uint32_t) * ncap));
            memcpy(nh, data(), sizeof(uint32_t) * n);
            free(heap); heap = nh; cap = ncap;
        }
        (heap ? heap : inl)[n++] = v;
    }
    const uint32_t* data() const { return heap ? heap : inl; }
    const uint32_t* begin() const { return data(); }
    const uint32_t* end() const { return data() + n; }
    size_t size() const { return n; }
    uint32_t operator[](size_t i) const { return data()[i]; }
};

struct pb2_htask_s {
    pb2_taskpool_t* tp = nullptr;
    pb2_task_class_t* tc = nullptr;
    int32_t id = -1;
    int32_t priority = 0;
    int32_t locals[4] = {0, 0, 0, 0};
    int nb_flows = 0;
    pb2_data_t* data[PB2_MAX_FLOWS] = {nullptr, nullptr, nullptr, nullptr};
    pb2_data_copy_t* data_in[PB2_MAX_FLOWS] = {nullptr, nullptr, nullptr, nullptr};
    pb2_data_copy_t* data_out[PB2_MAX_FLOWS] = {nullptr, nullptr, nullptr, nullptr};
    uint8_t access[PB2_MAX_FLOWS] = {0, 0, 0, 0};
    uint8_t pushout = 0;            // bit per flow, parsec_gpu_task_t::pushout
    bool use_mask = false;
    int32_t dep_goal = 0;           // counter: number of task-sourced inputs; mask: dependencies_goal
    int32_t dep_word = 0;           // counter: remaining; mask: satisfied bits
    int32_t npred_unsat = 0;        // unsatisfied in-edges
    pb2_succ_list succ;             // PB2_SUCC_MAKE(task id, dst flow)
    uint8_t body = 0;
    int32_t iparam[3] = {0, 0, 0};
    float fparam = 0.f;
    uint8_t chore_types = 0;
    uint8_t allowed_types = PB2_DEV_ANY_TYPE;   // DTD insert_task 'device' argument restricts the incarnations
    pb2_device_module_t* selected_device = nullptr;
    int64_t load = 0;
    uint8_t state = 0;              // 0 waiting, 1 queued ready, 2 owned by a device, 3 done
    int32_t window_index = -1;      // index in the window being built / run
    int32_t inwin_pred = 0;
    uint32_t seen_version[PB2_MAX_FLOWS] = {0, 0, 0, 0};
    uint64_t result = 0;
    int8_t ran_on = -1;
    // device_engine_trace: the window's time stamps of the task (its device's clock) and the SM; 0 when it ran elsewhere
    uint64_t dev_t_start = 0, dev_t_end = 0;
    uint32_t dev_smid = 0;
};

struct pb2_gpu_task_s {             // parsec_gpu_task_t, device_gpu.h:117-143
    uint16_t task_type = 0;         // PARSEC_GPU_TASK_TYPE_KERNEL
    uint16_t pushout = 0;
    int32_t last_status = 0;
    pb2_htask_t* ec = nullptr;
    uint32_t nb_flows = 0;
    size_t flow_span[PB2_MAX_FLOWS] = {0, 0, 0, 0};
};

struct pb2_dtd_tile_s {
    pb2_data_t* data = nullptr;
    int32_t last_writer = -1;               // task id, insert_function_internal.h:174-194
    std::vector<int32_t> readers_since;     // readers inserted since last_writer
    bool flushed = false;
};

// Tasks of a pool: stable addresses, id == index, allocated in chunks of 2048 (a std::deque of 270-byte elements does
// one malloc per task).
struct pb2_task_store {
    static constexpr size_t kChunk = 2048;
    std::vector<pb2_htask_s*> chunks;
    size_t n = 0;
    pb2_task_store() = default;
    pb2_task_store(const pb2_task_store&) = delete;
    pb2_task_store& operator=(const pb2_task_store&) = delete;
    ~pb2_task_store() { for (pb2_htask_s* c : chunks) delete[] c; }
    pb2_htask_s& emplace_back() {
        if (n == chunks.size() * kChunk) chunks.push_back(new pb2_htask_s[kChunk]);
        ++n;
        return back();
    }
    pb2_htask_s& operator[](size_t i) { return chunks[i / kChunk][i % kChunk]; }
    const pb2_htask_s& operator[](size_t i) const { return chunks[i / kChunk][i % kChunk]; }
    pb2_htask_s& back() { return (*this)[n - 1]; }
    size_t size() const { return n; }
};

struct pb2_taskpool_s {
    pb2_context_t* ctx = nullptr;
    int type = 0;                            // 0 DTD, 1 PTG
    std::string name;
    pb2_task_store tasks;                    // stable addresses; id == index
    std::deque<pb2_task_class_s> classes;
    std::vector<pb2_data_t*> temporaries;    // NEW data owned by the pool
    int32_t nb_done = 0;
    bool added = false;
    std::vector<int32_t> trace_task, trace_device;
    // device_engine_trace: the part records of the entities its tasks led (task = pool task id) and their device index
    std::vector<pb2_part_trace_t> part_trace;
    std::vector<int32_t> part_trace_device;
    std::map<std::pair<pb2_data_collection_t*, uint64_t>, pb2_dtd_tile_t*> tiles;
    std::vector<pb2_dtd_tile_t*> tile_list;
    uint32_t devices_index_mask = 0xffffffffu;
    std::function<void()> on_complete;       // PTG: final checks (e.g. CHECK task of pingpong)
};

struct pb2_device_window;                    // a window of the GPU device module, private to pb2_device_module.cpp

struct pb2_device_module_s {
    pb2_context_t* ctx = nullptr;
    std::string name;
    uint8_t device_index = 0, type = 0;
    int cuda_index = -1;
    int major = 0, minor = 0;
    bool dry_run = false;
    bool trace = false;                      // device_engine_trace at init: windows are created traced
    bool linked = false;                     // pb2_device_link_bodies: windows may run linked bodies
    bool linked_gemm = false;                // ... with PB2_LINK_GEMM_WINDOWS: GEMM windows too
    uint32_t linked_readers = 0;             // ... PB2_LINK_READERS: bit i, PB2_BODY_LINKED_0 + i is a reader
    uint32_t linked_gemm_bodies = 0;         // ... PB2_LINK_GEMM_BODIES: bit i, PB2_BODY_LINKED_0 + i runs in GEMM windows only
    bool linked_gemm_body_entry = false;     // ... PB2_LINK_GEMM_BODY_ENTRY: those run through pb2_linked_gemm_body
    int32_t gemm_body_parts[8] = {1, 1, 1, 1, 1, 1, 1, 1};   // pb2_device_set_gemm_body_parts, per GEMM-worker body
    pb2_engine_t* engine = nullptr;
    std::deque<pb2_device_window*> inflight; // windows launched and not yet retired (oldest first), pb2_device_module.cpp
    size_t pipe_chunk = 0;                   // roots per window while a large batch of pending tasks is being cut up
    pb2_device_stats_t st{};
    uint32_t peer_access_mask = 0;
    // memory: one slab carved by the zone heap (parsec_device_memory_reserve, device_gpu.c:866-991)
    void* slab = nullptr;
    size_t mem_block_size = 0;
    int64_t mem_nb_blocks = 0;
    pb2_zone zone;
    // the two LRUs (device_gpu.h:273-274), intrusive lists through pb2_data_copy_t::lru_prev/next
    pb2_data_copy_t *lru_head[3] = {nullptr, nullptr, nullptr}, *lru_tail[3] = {nullptr, nullptr, nullptr};
    int lru_count[3] = {0, 0, 0};
    std::deque<pb2_gpu_task_t*> pending;     // parsec_fifo_t pending
    int32_t mutex = 0;
    std::map<void*, void*> host_alias;       // registered host base -> device alias (non-collection memory)
};

struct pb2_context_s {
    int nb_cores = 1;
    std::vector<pb2_device_module_t*> devices;
    bool devices_frozen = false;
    std::map<std::string, int64_t> mca;
    std::vector<pb2_taskpool_t*> taskpools;
    std::vector<pb2_htask_t*> ready;         // priority-sorted ready list (parsec_list_push_sorted)
    size_t ready_head = 0;                   // entries before it have been handed out (pb2_context_wait)
    bool started = false;
    std::string last_error;
};

// ---- internal entry points shared by the translation units
pb2_htask_t* pb2i_new_task(pb2_taskpool_t* tp, pb2_task_class_t* tc);
void pb2i_add_edge(pb2_taskpool_t* tp, int32_t src, int32_t dst, int dst_flow);
void pb2i_schedule(pb2_context_t* ctx, pb2_htask_t* t);
int  pb2i_complete_execution(pb2_context_t* ctx, pb2_htask_t* t, int device_index);
int64_t pb2i_time_estimate(pb2_htask_t* t, pb2_device_module_t* d);
void pb2i_lru_remove(pb2_device_module_t* dev, pb2_data_copy_t* c);
void pb2i_lru_push_back(pb2_device_module_t* dev, int list, pb2_data_copy_t* c);
pb2_data_copy_t* pb2i_host_copy(pb2_data_t* d);
void* pb2i_device_visible_host_ptr(pb2_device_module_t* dev, pb2_data_t* data);
// the GPU device module (pb2_device_module.cpp): one step of a module with pending or in-flight windows (launch what
// is pending, retire the oldest window), and the end of every window still in flight, for pb2_fini
int  pb2i_device_progress(pb2_device_module_t* dev);
void pb2i_device_drain(pb2_device_module_t* dev);

// PB2_TIMING=1: the runtime reports on stderr where the host time of a wait goes
inline const bool pb2i_timing = getenv("PB2_TIMING") != nullptr;
inline double pb2i_now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
