// pb2_window_plan.hpp -- the host plan of an engine window: what pb2_window_create uploads and keeps, computed from the
// window's DAG and the engine's settings alone.  Host-only C++ (no CUDA type or call), so the rules it applies -- read
// groups, fused producers, GEMM units, parts, priority lanes, part records -- can be checked without a device.
#pragma once
#include <stdint.h>
#include <vector>
#include "pb2_window_layout.h"

namespace pb2 {

// What the engine hands the planner instead of itself.
struct PlanParams {
    int kind = 0;                         // 0: HBM bodies, 1: GEMM bodies
    bool shared = false;                  // pb2_engine_set_shared_windows
    bool trace = false;                   // pb2_engine_set_window_trace
    bool linked_image = false;            // the engine has linked an image (pb2_engine_link_bodies)
    bool linked_gemm = false;             // ... with PB2_LINK_GEMM_WINDOWS: linked bodies may run in GEMM windows too
    int queue_policy = 0, gemm_mode = 0, read_groups = 0, fuse_readers = 0;     // pb2_engine_params_t
    int nworkers = 1, nworkers_gemm = 1;
    int32_t part_bytes = 0, stage_slice_bytes = 0;
    uint32_t linked_sliceable = 0;        // bit i: PB2_BODY_LINKED_0 + i may be cut into parts
    uint32_t linked_checked = 0;          // bit i: PB2_BODY_LINKED_0 + i has a checked form (a subset of linked_sliceable)
    uint32_t linked_readers = 0;          // bit i: PB2_BODY_LINKED_0 + i is a reader (a subset of linked_sliceable)
    uint32_t linked_reader_groups = 0;    // bit i: reader PB2_BODY_LINKED_0 + i has the group form (a subset of linked_readers)
    uint32_t linked_gemm_bodies = 0;      // bit i: PB2_BODY_LINKED_0 + i gets the GEMM worker's operand ring (disjoint from
                                          // linked_sliceable)
    int32_t gemm_body_parts[8] = {1, 1, 1, 1, 1, 1, 1, 1};   // parts per task of GEMM-worker body PB2_BODY_LINKED_0 + i
    const int32_t* next_rs_begin = nullptr;     // shared windows: remote out-degree CSR (not owned)
};

// What every copy of a window's per-run state is sized from besides ntasks and ntiles.
struct RunShape {
    uint32_t ring = 0;                    // ring slots, a power of two
    int32_t nunits = 0;                   // GEMM windows: units
    bool parts = false;                   // per-task part counts (an HBM window with wide tasks)
    bool claims = false;                  // stage-in is sliced: claim arrays per tile
    bool lanes = false;                   // queue_policy 1: priority lanes, which start as lane_image
    bool trace = false;                   // part records (pb2_engine_set_window_trace)
    int32_t part_records = 0;             // trace: one part record per ring entry of a run
    Lanes lane_image{};
};

// Traced windows: a ring-entry owner that leads the entity of task `lead`, and where its nparts records start.
struct PartEntity { int32_t lead, base, nparts; };

// Everything pb2_window_create uploads or keeps, as host data.  An entry owner is a task of an HBM window or a unit of a
// GEMM window.
struct WindowPlan {
    std::vector<pb2_task_t> tasks;        // the device descriptors: flags masked (+ PB2_TASK_READER, _GROUP, PB2_TASK_GEMM_BODY), out-edges rewritten by read groups
    std::vector<uint32_t> succ;           // the device CSR
    std::vector<uint32_t> group;          // HBM windows with read groups (else empty): WinDev::group, group_mem
    std::vector<int32_t> group_mem;
    std::vector<uint16_t> nparts;         // HBM windows with wide tasks: parts per task (empty: every task is one part)
    std::vector<GUnit> units;             // GEMM windows: units, their members and their out-edges (unit ids)
    std::vector<GSeg> segs;
    std::vector<int32_t> usucc;
    std::vector<uint8_t> lane;            // queue_policy 1: per owner, its lane
    std::vector<int32_t> part_base;       // traced windows: per owner, its first part record
    std::vector<int32_t> ring_image;      // the first ring slots the reset kernel writes
    std::vector<int32_t> operand_rows, operand_inner;   // GEMM windows: tensor-map shape per tile (0: not an operand)
    RunShape run;
    int32_t slice_bytes = 0;              // stage-in slice size (WinDev::part_bytes)
    int32_t nlanes = 0;                   // queue_policy 1: lanes in use
    bool linked = false;                  // a task names a linked body: the window runs the engine's linked kernel of its kind
    std::vector<int32_t> task_entry;      // per task: its ring entry with (parts - 1) in the part field
    std::vector<int32_t> task_unit;       // traced windows, per task: the task that leads its scheduling entity
    std::vector<PartEntity> part_entities;     // traced windows: the ring-entry owners by leading task, their records
};

// The plan of a window of kind p.kind over the given DAG (the arguments of pb2_window_create, pointers non-null where
// their counts are positive).  Returns PB2_SUCCESS, or the error code with *why set to its message (left unchanged
// for the argument errors that have none).
int plan_window(const PlanParams& p, const pb2_task_t* tasks, int32_t ntasks, const uint32_t* succ, int32_t nsucc,
                const pb2_tile_t* tiles, int32_t ntiles, const int32_t* ready, int32_t nready, WindowPlan& plan,
                const char** why);

}  // namespace pb2
