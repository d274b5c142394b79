// Test-only C entry point to the window planner for tests/test_gemm_worker_bodies.py: wp_plan of window_plan_shim.cpp
// (built into the same library, which also gives wp_array, wp_scalar and wp_free) with PlanParams::linked_checked,
// linked_readers and linked_gemm_bodies as well, and linked_gemm set with linked_image (an engine linked with
// PB2_LINK_GEMM_WINDOWS).
#include "pb2_window_plan.hpp"

using namespace pb2;

extern "C" {

// prm as for wp_plan; linked_checked, linked_readers, linked_gemm_bodies: bit i, PB2_BODY_LINKED_0 + i has a checked
// form / is a reader / is a GEMM-worker body.
void* wp_plan_gemm_bodies(const int64_t* prm, uint32_t linked_checked, uint32_t linked_readers, uint32_t linked_gemm_bodies,
                          const pb2_task_t* tasks, int32_t ntasks, const uint32_t* succ, int32_t nsucc,
                          const pb2_tile_t* tiles, int32_t ntiles, const int32_t* ready, int32_t nready, int* rc,
                          const char** why) {
    PlanParams p;
    p.kind = (int)prm[0]; p.shared = prm[1] != 0; p.trace = prm[2] != 0; p.linked_image = p.linked_gemm = prm[3] != 0;
    p.queue_policy = (int)prm[4]; p.gemm_mode = (int)prm[5]; p.read_groups = (int)prm[6]; p.fuse_readers = (int)prm[7];
    p.nworkers = (int)prm[8]; p.nworkers_gemm = (int)prm[9];
    p.part_bytes = (int32_t)prm[10]; p.stage_slice_bytes = (int32_t)prm[11]; p.linked_sliceable = (uint32_t)prm[12];
    p.linked_checked = linked_checked; p.linked_readers = linked_readers; p.linked_gemm_bodies = linked_gemm_bodies;
    WindowPlan* plan = new WindowPlan();
    *why = nullptr;
    *rc = plan_window(p, tasks, ntasks, succ, nsucc, tiles, ntiles, ready, nready, *plan, why);
    if (*rc != PB2_SUCCESS) { delete plan; return nullptr; }
    return plan;
}

}  // extern "C"
