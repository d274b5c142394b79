// Test-only C entry points to the window planner (parsec_b200/csrc/pb2_window_plan.cpp) for tests/test_window_plan.py,
// which builds this file with g++ and no CUDA include path.
#include <string.h>
#include "pb2_window_plan.hpp"

using namespace pb2;

extern "C" {

// prm: kind, shared, trace, linked_image, queue_policy, gemm_mode, read_groups, fuse_readers, nworkers, nworkers_gemm,
// part_bytes, stage_slice_bytes, linked_sliceable.  Returns the plan (free it with wp_free), or null with *rc and *why
// set when plan_window refuses the window.
void* wp_plan(const int64_t* prm, const int32_t* next_rs_begin, const pb2_task_t* tasks, int32_t ntasks,
              const uint32_t* succ, int32_t nsucc, const pb2_tile_t* tiles, int32_t ntiles, const int32_t* ready,
              int32_t nready, int* rc, const char** why) {
    PlanParams p;
    p.kind = (int)prm[0]; p.shared = prm[1] != 0; p.trace = prm[2] != 0; p.linked_image = prm[3] != 0;
    p.queue_policy = (int)prm[4]; p.gemm_mode = (int)prm[5]; p.read_groups = (int)prm[6]; p.fuse_readers = (int)prm[7];
    p.nworkers = (int)prm[8]; p.nworkers_gemm = (int)prm[9];
    p.part_bytes = (int32_t)prm[10]; p.stage_slice_bytes = (int32_t)prm[11]; p.linked_sliceable = (uint32_t)prm[12];
    p.next_rs_begin = next_rs_begin;
    WindowPlan* plan = new WindowPlan();
    *why = nullptr;
    *rc = plan_window(p, tasks, ntasks, succ, nsucc, tiles, ntiles, ready, nready, *plan, why);
    if (*rc != PB2_SUCCESS) { delete plan; return nullptr; }
    return plan;
}

void wp_free(void* plan) { delete static_cast<WindowPlan*>(plan); }

// The plan array `name`: its bytes, *data pointing at them; -1 for an unknown name.
int64_t wp_array(const void* plan, const char* name, const void** data) {
    const WindowPlan& w = *static_cast<const WindowPlan*>(plan);
    auto out = [&](const auto& v) { *data = v.data(); return (int64_t)(v.size() * sizeof(v[0])); };
    if (!strcmp(name, "tasks")) return out(w.tasks);
    if (!strcmp(name, "succ")) return out(w.succ);
    if (!strcmp(name, "group")) return out(w.group);
    if (!strcmp(name, "group_mem")) return out(w.group_mem);
    if (!strcmp(name, "nparts")) return out(w.nparts);
    if (!strcmp(name, "units")) return out(w.units);
    if (!strcmp(name, "segs")) return out(w.segs);
    if (!strcmp(name, "usucc")) return out(w.usucc);
    if (!strcmp(name, "lane")) return out(w.lane);
    if (!strcmp(name, "part_base")) return out(w.part_base);
    if (!strcmp(name, "ring_image")) return out(w.ring_image);
    if (!strcmp(name, "operand_rows")) return out(w.operand_rows);
    if (!strcmp(name, "operand_inner")) return out(w.operand_inner);
    if (!strcmp(name, "task_entry")) return out(w.task_entry);
    if (!strcmp(name, "task_unit")) return out(w.task_unit);
    if (!strcmp(name, "part_entities")) return out(w.part_entities);
    if (!strcmp(name, "lane_begin")) { *data = w.run.lane_image.begin; return (int64_t)sizeof w.run.lane_image.begin; }
    if (!strcmp(name, "lane_ninit")) { *data = w.run.lane_image.ninit; return (int64_t)sizeof w.run.lane_image.ninit; }
    return -1;
}

// The plan scalar `name`; -1 for an unknown name.
int64_t wp_scalar(const void* plan, const char* name) {
    const WindowPlan& w = *static_cast<const WindowPlan*>(plan);
    if (!strcmp(name, "slice_bytes")) return w.slice_bytes;
    if (!strcmp(name, "nlanes")) return w.nlanes;
    if (!strcmp(name, "linked")) return w.linked;
    if (!strcmp(name, "ring")) return w.run.ring;
    if (!strcmp(name, "nunits")) return w.run.nunits;
    if (!strcmp(name, "parts")) return w.run.parts;
    if (!strcmp(name, "claims")) return w.run.claims;
    if (!strcmp(name, "lanes")) return w.run.lanes;
    if (!strcmp(name, "trace")) return w.run.trace;
    if (!strcmp(name, "part_records")) return w.run.part_records;
    return -1;
}

}  // extern "C"
