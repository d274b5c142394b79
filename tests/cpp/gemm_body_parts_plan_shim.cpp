// Test-only C entry point to the window planner for tests/test_gemm_body_parts.py: wp_plan_gemm_bodies of
// gemm_body_plan_shim.cpp (built into the same library with window_plan_shim.cpp, which gives wp_array, wp_scalar and
// wp_free) with PlanParams::gemm_body_parts as well.
#include "pb2_window_plan.hpp"

using namespace pb2;

extern "C" {

// prm, linked_checked, linked_readers, linked_gemm_bodies as for wp_plan_gemm_bodies; parts[i]: the part count of
// GEMM-worker body PB2_BODY_LINKED_0 + i (pb2_engine_set_gemm_body_parts).
void* wp_plan_gemm_body_parts(const int64_t* prm, uint32_t linked_checked, uint32_t linked_readers, uint32_t linked_gemm_bodies,
                              const int32_t* parts, const pb2_task_t* tasks, int32_t ntasks, const uint32_t* succ,
                              int32_t nsucc, const pb2_tile_t* tiles, int32_t ntiles, const int32_t* ready, int32_t nready,
                              int* rc, const char** why) {
    PlanParams p;
    p.kind = (int)prm[0]; p.shared = prm[1] != 0; p.trace = prm[2] != 0; p.linked_image = p.linked_gemm = prm[3] != 0;
    p.queue_policy = (int)prm[4]; p.gemm_mode = (int)prm[5]; p.read_groups = (int)prm[6]; p.fuse_readers = (int)prm[7];
    p.nworkers = (int)prm[8]; p.nworkers_gemm = (int)prm[9];
    p.part_bytes = (int32_t)prm[10]; p.stage_slice_bytes = (int32_t)prm[11]; p.linked_sliceable = (uint32_t)prm[12];
    p.linked_checked = linked_checked; p.linked_readers = linked_readers; p.linked_gemm_bodies = linked_gemm_bodies;
    for (int i = 0; i < 8; ++i) p.gemm_body_parts[i] = parts[i];
    WindowPlan* plan = new WindowPlan();
    *why = nullptr;
    *rc = plan_window(p, tasks, ntasks, succ, nsucc, tiles, ntiles, ready, nready, *plan, why);
    if (*rc != PB2_SUCCESS) { delete plan; return nullptr; }
    return plan;
}

}  // extern "C"
