// pb2_window_plan.cpp -- the host plan of an engine window (pb2_window_plan.hpp): argument checks, read groups and fused
// producers, units of GEMM windows, parts, priority lanes and the ring image, part records.
#include <string.h>
#include <algorithm>
#include <functional>
#include <utility>

#include "pb2_window_plan.hpp"

namespace pb2 {

namespace {

// What the ring plan knows of each initial ready-ring entry (plan.ring_image, in FIFO order) and of each entry owner.
struct Owners {
    std::vector<int32_t> entry_owner;     // the owner of each initial entry
    std::vector<uint32_t> pushes;         // queue_policy 1: per owner, the entries it can ever push
    uint32_t ring_slots = 0;              // ring slots the window needs besides the workers' slack
};

int validate_window(const PlanParams& p, const pb2_task_t* tasks, int32_t ntasks, const uint32_t* succ, int32_t nsucc,
                    int32_t ntiles, const int32_t* ready, int32_t nready, const char** why) {
    const int kind = p.kind;
    if (ntasks < 0 || nsucc < 0 || ntiles < 0 || nready < 0) return PB2_ERR_BAD_PARAM;
    if (kind != 0 && kind != 1) { *why = "window kind must be 0 (HBM bodies) or 1 (GEMM bodies)"; return PB2_ERR_BAD_PARAM; }
    if (ntasks >= (1 << 27)) return PB2_ERR_VALUE_OUT_OF_BOUNDS;
    // ready-ring entries of the HBM kernel carry the task id in 22 bits (PB2_ENT_MAKE: part << 22 | task)
    if (kind == 0 && ntasks >= (1 << 22)) { *why = "an HBM window holds at most 4194303 tasks (22-bit task id in the ready ring)"; return PB2_ERR_VALUE_OUT_OF_BOUNDS; }
    for (int32_t i = 0; i < ntasks; ++i) {
        const pb2_task_t& t = tasks[i];
        if (t.nb_flows > PB2_MAX_FLOWS) { *why = "task with more than PB2_MAX_FLOWS flows"; return PB2_ERR_BAD_PARAM; }
        if (t.succ_count < 0 || t.succ_begin < 0 || (int64_t)t.succ_begin + t.succ_count > nsucc) {
            *why = "successor range out of bounds"; return PB2_ERR_VALUE_OUT_OF_BOUNDS; }
        for (int f = 0; f < t.nb_flows; ++f)
            if (t.tile[f] >= ntiles) { *why = "tile id out of bounds"; return PB2_ERR_VALUE_OUT_OF_BOUNDS; }
        if (t.body >= PB2_BODY_MAX || t.body == PB2_BODY_USER) { *why = "unknown body id"; return PB2_ERR_BAD_PARAM; }
        if (kind == 0 && t.body == PB2_BODY_GEMM_BF16) {
            *why = "GEMM body in an HBM-kind window (use kind 1)"; return PB2_ERR_BAD_PARAM; }
        if (is_linked_body(t.body)) {
            const char* no = kind != 0 && !p.linked_gemm ? "linked body in a GEMM window (linked bodies run in HBM windows only)"
                           : p.shared ? "linked body in a shared window (not supported)"
                           : !p.linked_image ? "linked body id, but the engine has not linked an image (pb2_engine_link_bodies)"
                           : nullptr;
            if (no) { *why = no; return PB2_ERR_NOT_SUPPORTED; }
            if (kind == 0 && ((p.linked_gemm_bodies >> (t.body - PB2_BODY_LINKED_0)) & 1u)) {
                *why = "GEMM-worker body in an HBM window (it runs in GEMM windows only, on the worker's operand ring)";
                return PB2_ERR_NOT_SUPPORTED;
            }
        }
    }
    for (int32_t i = 0; i < nsucc; ++i)
        if (PB2_SUCC_TASK(succ[i]) >= ntasks) { *why = "successor id out of bounds"; return PB2_ERR_VALUE_OUT_OF_BOUNDS; }
    for (int32_t i = 0; i < nready; ++i)
        if (ready[i] < 0 || ready[i] >= ntasks) { *why = "ready id out of bounds"; return PB2_ERR_VALUE_OUT_OF_BOUNDS; }
    return PB2_SUCCESS;
}

// GEMM windows: one tensor map per tile used as an operand, [rows][inner] bf16 (pb2_window_create encodes them).  The
// shape of each operand tile, checked against every GEMM task that reads it and against the tile's bytes.
int plan_gemm_operands(const pb2_task_t* tasks, int32_t ntasks, const pb2_tile_t* tiles, int32_t ntiles,
                       WindowPlan& plan, const char** why) {
    std::vector<int32_t>& rows = plan.operand_rows;
    std::vector<int32_t>& inner = plan.operand_inner;
    rows.assign((size_t)ntiles, 0); inner.assign((size_t)ntiles, 0);
    for (int32_t i = 0; i < ntasks; ++i) {
        const pb2_task_t& t = tasks[i];
        if (t.body != PB2_BODY_GEMM_BF16) continue;
        if (t.nb_flows < 3 || t.tile[0] < 0 || t.tile[1] < 0 || t.tile[2] < 0) { *why = "GEMM task needs 3 data flows"; return PB2_ERR_BAD_PARAM; }
        const int M = t.iparam[0], N = t.iparam[1], K = t.iparam[2];
        if (M <= 0 || N <= 0 || K <= 0 || (K % 8) || (N % 8)) { *why = "GEMM tile: need M,N,K > 0, K % 8 == 0, N % 8 == 0"; return PB2_ERR_NOT_SUPPORTED; }
        const int32_t need[2][2] = {{M, K}, {N, K}};
        for (int f = 0; f < 2; ++f) {
            const int32_t id = t.tile[f];
            if (rows[id] == 0) { rows[id] = need[f][0]; inner[id] = need[f][1]; }
            else if (rows[id] != need[f][0] || inner[id] != need[f][1]) { *why = "tile used with two different operand shapes"; return PB2_ERR_NOT_SUPPORTED; }
            if ((uint64_t)need[f][0] * need[f][1] * 2 > tiles[id].bytes) { *why = "GEMM operand larger than its tile"; return PB2_ERR_VALUE_OUT_OF_BOUNDS; }
        }
        if ((uint64_t)M * N * 2 > tiles[t.tile[2]].bytes) { *why = "GEMM C larger than its tile"; return PB2_ERR_VALUE_OUT_OF_BOUNDS; }
    }
    return PB2_SUCCESS;
}

// Every body but NOP loads and stores its tiles' slots with 16-byte vectors (GEMM operands through TMA): a slot of such a
// task must be 16-byte aligned, or the window would fault instead of failing here.  Empty tiles are never accessed.
int check_slot_alignment(const pb2_task_t* tasks, int32_t ntasks, const pb2_tile_t* tiles, const char** why) {
    for (int32_t i = 0; i < ntasks; ++i) {
        const pb2_task_t& t = tasks[i];
        if (t.body == PB2_BODY_NOP) continue;
        for (int f = 0; f < t.nb_flows; ++f) {
            const int32_t id = t.tile[f];
            if (id < 0 || tiles[id].bytes == 0 || !((uintptr_t)tiles[id].dev_ptr & 15)) continue;
            *why = t.body == PB2_BODY_GEMM_BF16 ? "GEMM tile not 16-byte aligned" : "tile of a task body not 16-byte aligned";
            return PB2_ERR_BAD_PARAM;
        }
    }
    return PB2_SUCCESS;
}

// ---------------------------------------------------------------------------------------------
// queue_policy 1: priority lanes
// ---------------------------------------------------------------------------------------------
// The lane of every task: the distinct priorities of the window's tasks ranked highest first, lane = rank r with at most
// PB2_PRIO_LANES of them, floor(r * PB2_PRIO_LANES / ndistinct) otherwise.  tests/priority_order.py restates it.
std::vector<uint8_t> task_priority_lanes(const pb2_task_t* tasks, int32_t ntasks, int32_t* nlanes) {
    std::vector<int32_t> v((size_t)ntasks);
    for (int32_t i = 0; i < ntasks; ++i) v[(size_t)i] = tasks[i].priority;
    std::sort(v.begin(), v.end(), std::greater<int32_t>());
    v.erase(std::unique(v.begin(), v.end()), v.end());
    const int64_t nd = (int64_t)v.size();
    std::vector<uint8_t> lane((size_t)ntasks, 0);
    for (int32_t i = 0; i < ntasks; ++i) {
        const int64_t r = std::lower_bound(v.begin(), v.end(), tasks[i].priority, std::greater<int32_t>()) - v.begin();
        lane[(size_t)i] = (uint8_t)(nd <= PB2_PRIO_LANES ? r : r * PB2_PRIO_LANES / nd);
    }
    *nlanes = nd == 0 ? 1 : (int32_t)std::min<int64_t>(nd, PB2_PRIO_LANES);
    return lane;
}

// Cut the ring into one segment per lane, as long as the entries the lane's owners can ever push (owner o, in lane
// plan.lane[o], pushes at most o.pushes[o] entries).  plan.ring_image becomes the image of the whole ring that the
// reset kernel writes: each entry at the start of its owner's lane's segment, in the same order within a lane; the
// lanes start as plan.run.lane_image.
void build_lane_ring(WindowPlan& plan, const Owners& o) {
    Lanes& h = plan.run.lane_image;
    plan.run.lanes = true;
    uint32_t size[PB2_PRIO_LANES] = {0};
    for (size_t i = 0; i < plan.lane.size(); ++i) size[plan.lane[i]] += o.pushes[i];
    uint32_t b = 0;
    for (int l = 0; l < PB2_PRIO_LANES; ++l) { h.begin[l] = b; b += size[l]; }
    std::vector<int32_t> ring(b, kEmpty);
    for (size_t i = 0; i < plan.ring_image.size(); ++i) {
        const int l = plan.lane[(size_t)o.entry_owner[i]];
        ring[h.begin[l] + h.ninit[l]++] = plan.ring_image[i];
    }
    plan.ring_image.swap(ring);
}

// Traced windows: where the part records of each ring-entry owner o (a task of an HBM window, a unit of a GEMM window)
// start.  Owner o leads the entity of task lead[o] and runs nparts[o] parts (0: o owns no entries, as the members of a
// read group).  Its records are part_base[o] .. + nparts[o], in owner order; pb2_window_part_trace returns them by
// leading task.
void plan_part_records(const std::vector<int32_t>& lead, const std::vector<int32_t>& nparts, WindowPlan& plan) {
    std::vector<int32_t>& base = plan.part_base;
    base.resize(nparts.size());
    int32_t n = 0;
    plan.part_entities.clear();
    for (size_t o = 0; o < nparts.size(); ++o) {
        base[o] = n;
        if (nparts[o] > 0) plan.part_entities.push_back({lead[o], n, nparts[o]});
        n += nparts[o];
    }
    std::stable_sort(plan.part_entities.begin(), plan.part_entities.end(),
                     [](const PartEntity& a, const PartEntity& b) { return a.lead < b.lead; });
    plan.run.part_records = n;
}

// ---------------------------------------------------------------------------------------------
// GEMM windows: group tasks into units (fused k-chains), see pb2_gemm.cuh
// ---------------------------------------------------------------------------------------------
// The plan of a GEMM window: its units are the ring-entry owners.  task_lane (queue_policy 1, else empty): a unit's
// lane is the lane of its first task, for all its parts.  A unit that runs an HBM body is cut into
// task_parts(..., kMaxParts) byte-slice parts, as HBM windows cut their wide tasks.  The window's read groups
// (plan.group, formed on plan.tasks and plan.succ before) are units of HBM bodies: a group's members in member order,
// the leader first, preceded by the producer when one runs with them (flag bit 2); its parts are the first task's.
int build_gemm2_units(const PlanParams& p, const pb2_task_t* tasks, int32_t ntasks, const uint32_t* succ,
                      const int32_t* ready, int32_t nready, bool fuse, const int32_t* rs_begin,
                      const std::vector<uint8_t>& task_lane, const pb2_tile_t* tiles, int32_t part_bytes,
                      WindowPlan& plan, Owners& own, const char** why) {
    std::vector<int32_t> indeg((size_t)ntasks, 0), cpred((size_t)ntasks, -1), ccons((size_t)ntasks, 0), next((size_t)ntasks, -1);
    auto is_gemm = [&](int32_t t) { return tasks[t].body == PB2_BODY_GEMM_BF16; };
    for (int32_t u = 0; u < ntasks; ++u)
        for (int32_t e = 0; e < tasks[u].succ_count; ++e) {
            const uint32_t s = succ[tasks[u].succ_begin + e];
            const int32_t t = PB2_SUCC_TASK(s);
            indeg[t]++;
            if (PB2_SUCC_FLOW(s) == 2 && is_gemm(u) && is_gemm(t) && tasks[u].tile[2] == tasks[t].tile[2]) { ccons[u]++; cpred[t] = u; }
        }
    // A window that peers release into: the tasks' dependency goals (counter mode, set by the partitioner) also
    // count the in-edges that come from other GPUs; the local CSR does not show them.
    if (p.shared)
        for (int32_t t = 0; t < ntasks; ++t) {
            const int32_t need = (tasks[t].flags & PB2_TASK_DEPS_MASK) ? __builtin_popcount((unsigned)tasks[t].dep_goal) : tasks[t].dep_goal;
            if (need < indeg[t]) { *why = "dependency goal smaller than the in-window in-degree"; return PB2_ERR_BAD_PARAM; }
            indeg[t] = need;
        }
    if (fuse)
        for (int32_t t = 0; t < ntasks; ++t) {
            const int32_t u = cpred[t];
            if (u < 0 || indeg[t] != 1 || ccons[u] != 1) continue;                 // the chain link must be t's only missing input
            if (rs_begin && rs_begin[u + 1] > rs_begin[u]) continue;               // u's result is awaited on another GPU: retire it on its own
            if (tasks[u].access[2] & PB2_FLOW_PUSHOUT) continue;                   // u's C has to reach the host: flush there
            if (memcmp(tasks[u].iparam, tasks[t].iparam, sizeof tasks[u].iparam)) continue;
            next[u] = t;
        }
    // a read group runs as one unit: its members follow its first task (a GEMM task is never in one, see fusable)
    for (int32_t t = 0; t < (int32_t)plan.group.size(); ++t) {
        const uint32_t gd = plan.group[(size_t)t];
        const int32_t* mem = plan.group_mem.data() + ((gd & ~PB2_GROUP_FUSED) >> 4);
        if (gd & PB2_GROUP_FUSED) next[(size_t)t] = mem[0];             // the producer, then the group it runs with
        else for (uint32_t i = 1; i < (gd & 15u); ++i) next[(size_t)mem[i - 1]] = mem[i];     // t leads the group
    }
    std::vector<uint8_t> has_pred((size_t)ntasks, 0);
    for (int32_t u = 0; u < ntasks; ++u) if (next[u] >= 0) has_pred[next[u]] = 1;
    std::vector<GUnit>& units = plan.units;
    std::vector<GSeg>& segs = plan.segs;
    std::vector<int32_t> unit_of((size_t)ntasks, -1);
    for (int32_t h = 0; h < ntasks; ++h) {
        if (has_pred[h]) continue;
        GUnit u{}; u.seg_begin = (int32_t)segs.size(); u.dep_goal = indeg[h];
        const bool g = is_gemm(h);
        u.flags = g ? 1 : 0; u.tileC = g ? tasks[h].tile[2] : -1;
        u.M = tasks[h].iparam[0]; u.N = tasks[h].iparam[1]; u.K = tasks[h].iparam[2];
        // a part runs every nparts-th 128 x 256 sub-tile of C, or one byte slice of the tiles of an HBM body; a linked
        // body whose sliceable bit is clear runs as one part over whole tiles, and a GEMM-worker body as the parts its
        // count declares, each over whole tiles (the body splits the work by part index itself)
        const bool whole = is_linked_body(tasks[h].body) && !((p.linked_sliceable >> (tasks[h].body - PB2_BODY_LINKED_0)) & 1u);
        u.nparts = g ? std::min(((u.M + gemm::BM - 1) / gemm::BM) * ((u.N + gemm::BN - 1) / gemm::BN), gemm::kMaxParts)
                 : (tasks[h].flags & PB2_TASK_GEMM_BODY) ? p.gemm_body_parts[tasks[h].body - PB2_BODY_LINKED_0]
                 : whole ? 1 : task_parts(tasks[h], [&](int32_t id) { return tiles[id].bytes; }, part_bytes, gemm::kMaxParts);
        if (!plan.group.empty() && (plan.group[(size_t)h] & PB2_GROUP_FUSED)) u.flags |= 4;
        for (int32_t t = h; t >= 0; t = next[t]) {
            unit_of[t] = (int32_t)units.size();
            segs.push_back(GSeg{t, g ? tasks[t].tile[0] : -1, g ? tasks[t].tile[1] : -1, 0});
            if (g && (tasks[t].access[2] & PB2_FLOW_PUSHOUT)) u.flags |= 2;
        }
        u.seg_count = (int32_t)segs.size() - u.seg_begin;
        units.push_back(u);
    }
    std::vector<int32_t>& usucc = plan.usucc;
    for (GUnit& u : units) {
        u.succ_begin = (int32_t)usucc.size();
        for (int32_t i = 0; i < u.seg_count; ++i) {
            const int32_t t = segs[u.seg_begin + i].task;
            for (int32_t e = 0; e < tasks[t].succ_count; ++e) {
                const int32_t d = PB2_SUCC_TASK(succ[tasks[t].succ_begin + e]);
                if (is_gemm(t) && d == next[t] && PB2_SUCC_FLOW(succ[tasks[t].succ_begin + e]) == 2) continue;   // the fused link
                usucc.push_back(unit_of[d]);
            }
        }
        u.succ_count = (int32_t)usucc.size() - u.succ_begin;
    }
    uint32_t total_parts = 0;
    for (const GUnit& u : units) total_parts += (uint32_t)u.nparts;
    // Ready GEMM units enter the ring in Z-order of their (locals[0], locals[1]) = C(i,j) coordinates: the units
    // that run concurrently then form a compact block of C tiles that shares A rows and B columns in L2 (a FIFO
    // ring keeps whatever order the host gives it; the reference's priority hint mt*nt*kt - i*nt + j plays the
    // same role for its sorted pending list, device_gpu.c:2169-2174).
    std::vector<std::pair<uint64_t, int32_t>> order;
    auto morton = [](uint32_t x, uint32_t y) {
        uint64_t r = 0;
        for (int b = 0; b < 16; ++b) r |= ((uint64_t)((x >> b) & 1) << (2 * b + 1)) | ((uint64_t)((y >> b) & 1) << (2 * b));
        return r;
    };
    for (int32_t i = 0; i < nready; ++i) {
        const int32_t uid = unit_of[ready[i]];
        if (units[uid].dep_goal != 0) { *why = "ready task has in-window predecessors"; return PB2_ERR_BAD_PARAM; }
        const pb2_task_t& t = tasks[ready[i]];
        const uint64_t key = (units[uid].flags & 1) ? morton((uint32_t)t.locals[0], (uint32_t)t.locals[1]) : 0;
        order.emplace_back(key, uid);
    }
    std::stable_sort(order.begin(), order.end(), [](const std::pair<uint64_t, int32_t>& a, const std::pair<uint64_t, int32_t>& b) { return a.first < b.first; });
    for (auto& o : order)
        for (int32_t q = 0; q < units[o.second].nparts; ++q) {
            plan.ring_image.push_back((int32_t)PB2_SUCC_MAKE(o.second, q));
            own.entry_owner.push_back(o.second);
        }
    if (!task_lane.empty())
        for (const GUnit& u : units) {
            plan.lane.push_back(task_lane[(size_t)segs[(size_t)u.seg_begin].task]);
            own.pushes.push_back((uint32_t)u.nparts);
        }
    own.ring_slots = (uint32_t)ntasks + total_parts;
    // operand tiles that have to be staged in (host or peer GPU) are pulled in 64 KiB slices by every worker
    // that needs them (the parts of one unit, the units that share an operand) instead of by one worker alone
    plan.slice_bytes = 64 * 1024;
    plan.run.claims = true;
    plan.run.nunits = (int32_t)units.size();
    plan.task_entry.resize((size_t)ntasks);
    for (int32_t t = 0; t < ntasks; ++t) plan.task_entry[(size_t)t] = (int32_t)PB2_SUCC_MAKE(unit_of[t], units[(size_t)unit_of[t]].nparts - 1);
    if (!plan.task_unit.empty()) {
        for (int32_t t = 0; t < ntasks; ++t) plan.task_unit[(size_t)t] = segs[(size_t)units[(size_t)unit_of[t]].seg_begin].task;
        std::vector<int32_t> lead(units.size()), np(units.size());
        for (size_t u = 0; u < units.size(); ++u) { lead[u] = segs[(size_t)units[u].seg_begin].task; np[u] = units[u].nparts; }
        plan_part_records(lead, np, plan);
    }
    return PB2_SUCCESS;
}

// ---------------------------------------------------------------------------------------------
// read groups
// ---------------------------------------------------------------------------------------------
// A run of >= 2 consecutive out-edges of one task whose targets all
//   - have that edge as their only input (in-degree 1, not ready at start; counter goal 1, or the edge's one mask bit),
//   - run a CHECK body over exactly one data flow, flow 0, READ only, on the same tile,
// becomes one edge to the run's first target (the leader) in the device CSR, and the leader's worker streams the tile
// once for all the members (pb2_engine_hbm_kernel).  Without groups F readers of a tile each pull it through L2 into
// their own SM, F passes where one carries the same bytes.  The members become ready together and would have entered
// the FIFO ring back to back: with one worker the retire order is the ungrouped one.  Runs longer than PB2_GROUP_MAX
// are split.  O(ntasks + nsucc); tasks keep their own out-edges.  Returns false when no group formed.
//
// With `fuse`, a task P also runs with the first group among its out-edges as one unit when P has a body, writes the
// group's tile X without pushing it out, and X is P's widest tile (so P's parts cut X as the members' parts do): the
// edge P -> leader leaves the device CSR and group[P] = PB2_GROUP_FUSED | the leader's group word.  The worker that
// runs a part of P writes it to X and checks every value for the members in registers before it stores it
// (run_fused_part); so P's body must have a checked form that writes X (fusable).  A linked body has one when its bit
// is set in `linked_checked` (pb2_engine_link_bodies_checked); X must then be the only tile P writes, since the kernel
// knows nothing else of what the body stores (run_linked_part).  The
// caller turns fusion off with one worker: there the retire order is the FIFO order, in which the members run after
// every task that was queued when P retired, and a fused unit runs them right after P.
//
// Linked readers (a body declared a reader, PB2_LINK_READERS; plan_window marks its tasks PB2_TASK_READER) are members
// under the same rules, in groups of their own: a run splits where CHECK members and linked readers meet, and a group's
// linked readers may run different bodies.  Their worker walks each part in chunks and calls every member on a chunk
// before the next one, so that the members re-read it from the SM's caches (run_linked_group_part).  A producer runs
// with such a group when it is a built-in fusable body, or a sliceable linked body that writes X and no other tile: it
// needs no checked form, as it writes each chunk before the members read it back.
bool form_read_groups(std::vector<pb2_task_t>& tasks, const uint32_t* succ, const int32_t* ready, int32_t nready,
                      const pb2_tile_t* tiles, bool fuse, const PlanParams& prm,
                      std::vector<uint32_t>& gsucc, std::vector<uint32_t>& group, std::vector<int32_t>& gmem) {
    const size_t n = tasks.size();
    std::vector<uint8_t> indeg(n, 0);                        // saturates at 2
    for (size_t u = 0; u < n; ++u)
        for (int32_t j = 0; j < tasks[u].succ_count; ++j) {
            uint8_t& d = indeg[(size_t)PB2_SUCC_TASK(succ[tasks[u].succ_begin + j])];
            if (d < 2) ++d;
        }
    for (int32_t i = 0; i < nready; ++i) indeg[(size_t)ready[i]] = 2;
    auto linked_bit = [](uint32_t mask, int body) { return is_linked_body(body) && ((mask >> (body - PB2_BODY_LINKED_0)) & 1u); };
    // the member kind of edge s's target: 0 none, 1 CHECK, 2 linked reader
    auto reader = [&](uint32_t s) {
        const pb2_task_t& t = tasks[(size_t)PB2_SUCC_TASK(s)];
        if (indeg[(size_t)PB2_SUCC_TASK(s)] != 1) return 0;
        if (t.dep_goal != ((t.flags & PB2_TASK_DEPS_MASK) ? (int32_t)(1u << PB2_SUCC_FLOW(s)) : 1)) return 0;
        const int kind = t.body == PB2_BODY_CHECK_I32 || t.body == PB2_BODY_CHECK_F32 ? 1 : (t.flags & PB2_TASK_READER) ? 2 : 0;
        if (!kind) return 0;
        if (t.nb_flows < 1 || t.tile[0] < 0 || (t.access[0] & (PB2_FLOW_ACCESS_RW | PB2_FLOW_PUSHOUT)) != PB2_FLOW_ACCESS_READ) return 0;
        for (int f = 1; f < t.nb_flows; ++f) if (t.tile[f] >= 0) return 0;
        return kind;
    };
    // the bodies with a checked form (run_hbm_body<true>), whose output flow `out` writes X; with linked readers
    // (kind 2) the built-in ones and the sliceable linked ones
    auto fusable = [&](const pb2_task_t& p, int32_t x, int kind) {
        if (is_linked_body(p.body)) {
            if (!linked_bit(kind == 2 ? prm.linked_sliceable : prm.linked_checked, p.body)) return false;
            int writes = 0;
            for (int f = 0; f < p.nb_flows; ++f) {
                if (p.tile[f] < 0) continue;
                if (tiles[p.tile[f]].bytes > tiles[x].bytes) return false;
                if (!(p.access[f] & PB2_FLOW_ACCESS_WRITE)) continue;
                if (p.tile[f] != x || (p.access[f] & PB2_FLOW_PUSHOUT)) return false;
                ++writes;
            }
            return writes == 1;
        }
        int out = 0;
        switch (p.body) {
        case PB2_BODY_FILL_I32: case PB2_BODY_FILL_F32: case PB2_BODY_MEMSET_U8: case PB2_BODY_INCR_I32:
        case PB2_BODY_SCALE_I32: case PB2_BODY_ADD_IOTA_I32: case PB2_BODY_IOTA_I32: case PB2_BODY_INCR_F32: break;
        case PB2_BODY_COPY: case PB2_BODY_AXPY_F32: out = 1; break;
        default: return false;
        }
        if (p.nb_flows <= out || p.tile[out] != x || !(p.access[out] & PB2_FLOW_ACCESS_WRITE)) return false;
        // the checked COPY / AXPY writes every byte of the slice: the tile they read is as long as X
        if (out == 1 && (p.tile[0] < 0 || tiles[p.tile[0]].bytes != tiles[x].bytes)) return false;
        for (int f = 0; f < p.nb_flows; ++f) {
            if (p.tile[f] < 0) continue;
            if (tiles[p.tile[f]].bytes > tiles[x].bytes) return false;
            if (p.tile[f] == x && (p.access[f] & PB2_FLOW_ACCESS_WRITE) && (p.access[f] & PB2_FLOW_PUSHOUT)) return false;
        }
        return true;
    };
    std::vector<int32_t> begin(n), count(n);
    group.assign(n, 0u);
    gsucc.clear(); gmem.clear();
    for (size_t u = 0; u < n; ++u) {
        const uint32_t* out = succ + tasks[u].succ_begin;
        const int32_t c = tasks[u].succ_count;
        begin[u] = (int32_t)gsucc.size();
        bool first_group = true;
        for (int32_t j = 0; j < c;) {
            int32_t r = j + 1;
            int32_t tile = -1;
            const int kind = reader(out[j]);
            if (kind) {
                tile = tasks[(size_t)PB2_SUCC_TASK(out[j])].tile[0];
                while (r < c && r - j < PB2_GROUP_MAX && reader(out[r]) == kind && tasks[(size_t)PB2_SUCC_TASK(out[r])].tile[0] == tile) ++r;
            }
            bool fused = false;
            if (r - j >= 2) {
                const uint32_t gw = ((uint32_t)gmem.size() << 4) | (uint32_t)(r - j);
                group[(size_t)PB2_SUCC_TASK(out[j])] = gw;
                for (int32_t q = j; q < r; ++q) gmem.push_back(PB2_SUCC_TASK(out[q]));
                fused = fuse && first_group && fusable(tasks[u], tile, kind);
                if (fused) group[u] = PB2_GROUP_FUSED | gw;
                first_group = false;
            }
            if (!fused) gsucc.push_back(out[j]);
            j = r;
        }
        count[u] = (int32_t)gsucc.size() - begin[u];
    }
    if (gmem.empty()) return false;
    for (size_t u = 0; u < n; ++u) { tasks[u].succ_begin = begin[u]; tasks[u].succ_count = count[u]; }
    return true;
}

// The read groups and fused producers of a window of either kind (form_read_groups), with the engine's settings:
// none in a shared window (it is released into by task id from other GPUs and pushes per task: its tasks run alone) or
// with read_groups < 0, no fusion with fuse_readers < 0 or with one worker of the window's kind (nworkers).  Rewrites
// the out-edges of plan.tasks and sets plan.succ, and plan.group and group_mem when a group formed (returns true then).
bool plan_read_groups(const PlanParams& p, int nworkers, const uint32_t* succ, int32_t nsucc, const pb2_tile_t* tiles,
                      const int32_t* ready, int32_t nready, WindowPlan& plan) {
    std::vector<uint32_t> gsucc, group;
    std::vector<int32_t> gmem;
    const bool grouped = !p.shared && p.read_groups >= 0 &&
                         form_read_groups(plan.tasks, succ, ready, nready, tiles, p.fuse_readers >= 0 && nworkers > 1,
                                          p, gsucc, group, gmem);
    if (grouped) { plan.succ.swap(gsucc); plan.group.swap(group); plan.group_mem.swap(gmem); }
    else plan.succ.assign(succ, succ + nsucc);
    return grouped;
}

// The plan of an HBM window: its tasks (plan.tasks) are the ring-entry owners, each cut into task_parts(...,
// PB2_MAX_PARTS) parts.  task_lane: as for build_gemm2_units.  Forms the read groups (plan_read_groups).
void plan_hbm_window(const PlanParams& p, const uint32_t* succ, int32_t nsucc, const pb2_tile_t* tiles, int32_t ntiles,
                     const int32_t* ready, int32_t nready, const std::vector<uint8_t>& task_lane, WindowPlan& plan,
                     Owners& own) {
    std::vector<pb2_task_t>& dtasks = plan.tasks;
    const int32_t ntasks = (int32_t)dtasks.size();
    std::vector<uint16_t> nparts((size_t)ntasks);
    uint32_t extra_parts = 0;
    plan.task_entry.resize((size_t)ntasks);
    for (int32_t i = 0; i < ntasks; ++i) {
        // a linked body whose sliceable bit is clear runs over whole tiles (a stencil reads its neighbours' tiles)
        const pb2_task_t& t = dtasks[(size_t)i];
        const bool whole = is_linked_body(t.body) && !((p.linked_sliceable >> (t.body - PB2_BODY_LINKED_0)) & 1u);
        const int np = whole ? 1 : task_parts(t, [&](int32_t id) { return tiles[id].bytes; }, p.part_bytes, PB2_MAX_PARTS);
        nparts[(size_t)i] = (uint16_t)np; extra_parts += (uint32_t)np - 1;
        plan.task_entry[(size_t)i] = PB2_ENT_MAKE(i, np - 1);
    }
    for (int32_t i = 0; i < nready; ++i)
        for (int q = 0; q < (int)nparts[(size_t)ready[i]]; ++q) {
            plan.ring_image.push_back(PB2_ENT_MAKE(ready[i], q));
            own.entry_owner.push_back(ready[i]);
        }
    if (!task_lane.empty()) { plan.lane = task_lane; own.pushes.assign(nparts.begin(), nparts.end()); }
    own.ring_slots = (uint32_t)ntasks + extra_parts;
    // Stage-in is cut finer than tasks are: a tile that has to come from the host or a peer GPU is pulled in slices
    // by EVERY worker that needs it (claim bit per slice), so the readers of a tile share the transfer instead of one
    // moving it while the others wait.
    plan.slice_bytes = stage_slice(p.stage_slice_bytes, p.part_bytes);
    plan.run.parts = plan.run.claims = extra_parts > 0;
    for (int32_t i = 0; i < ntiles && !plan.run.claims; ++i)
        plan.run.claims = plan.slice_bytes > 0 && tiles[i].state != PB2_TILE_VALID && tiles[i].bytes > (uint32_t)plan.slice_bytes;
    if (plan_read_groups(p, p.nworkers, succ, nsucc, tiles, ready, nready, plan)) {
        // a read group is led by its leader, unless a producer runs with it: then by the producer
        if (!plan.task_unit.empty())
            for (int pass = 0; pass < 2; ++pass)
                for (int32_t t = 0; t < ntasks; ++t) {
                    const uint32_t gd = plan.group[(size_t)t];
                    if ((gd & 15u) == 0 || ((gd & PB2_GROUP_FUSED) != 0) != (pass == 1)) continue;
                    const uint32_t b = (gd & ~PB2_GROUP_FUSED) >> 4;
                    for (uint32_t i = 0; i < (gd & 15u); ++i) plan.task_unit[(size_t)plan.group_mem[b + i]] = t;
                }
    }
    if (!plan.task_unit.empty()) {                // a task owns ring entries unless a group member is led by another task
        std::vector<int32_t> lead((size_t)ntasks), np((size_t)ntasks);
        for (int32_t t = 0; t < ntasks; ++t) { lead[(size_t)t] = t; np[(size_t)t] = plan.task_unit[(size_t)t] == t ? nparts[(size_t)t] : 0; }
        plan_part_records(lead, np, plan);
    }
    if (extra_parts) plan.nparts.swap(nparts);
}

}  // namespace

int plan_window(const PlanParams& p, const pb2_task_t* tasks, int32_t ntasks, const uint32_t* succ, int32_t nsucc,
                const pb2_tile_t* tiles, int32_t ntiles, const int32_t* ready, int32_t nready, WindowPlan& plan,
                const char** why) {
    int rc = validate_window(p, tasks, ntasks, succ, nsucc, ntiles, ready, nready, why);
    if (rc != PB2_SUCCESS) return rc;
    if ((rc = check_slot_alignment(tasks, ntasks, tiles, why)) != PB2_SUCCESS) return rc;
    const bool prio = p.queue_policy == 1;
    if (prio && p.shared) {
        *why = "queue_policy 1 (priority lanes) is not supported with shared windows: peers push into one FIFO ring";
        return PB2_ERR_NOT_SUPPORTED;
    }
    plan = WindowPlan{};
    plan.tasks.assign(tasks, tasks + ntasks);
    for (pb2_task_t& t : plan.tasks) {
        t.flags &= 0x07;
        if (is_linked_body(t.body)) {
            plan.linked = true;
            if ((p.linked_readers >> (t.body - PB2_BODY_LINKED_0)) & 1u) t.flags |= PB2_TASK_READER;
            if ((p.linked_reader_groups >> (t.body - PB2_BODY_LINKED_0)) & 1u) t.flags |= PB2_TASK_READER_GROUP;
            // a GEMM-worker body is not sliceable (link_args_error): its task runs as one part, is never a reader and
            // never a fused producer (form_read_groups), so it always runs alone on its worker, with the whole ring
            if ((p.linked_gemm_bodies >> (t.body - PB2_BODY_LINKED_0)) & 1u) t.flags |= PB2_TASK_GEMM_BODY;
        }
    }
    std::vector<uint8_t> task_lane;
    if (prio) task_lane = task_priority_lanes(tasks, ntasks, &plan.nlanes);
    if (p.trace) {                              // every task leads itself until a plan groups it
        plan.task_unit.resize((size_t)ntasks);
        for (int32_t t = 0; t < ntasks; ++t) plan.task_unit[(size_t)t] = t;
    }
    plan.run.trace = p.trace;
    Owners own;
    if (p.kind == 0) plan_hbm_window(p, succ, nsucc, tiles, ntiles, ready, nready, task_lane, plan, own);
    else {
        // HBM bodies of a GEMM window are cut into parts as HBM windows cut them.  Not in shared windows: their units
        // are released by peers over NVLink, and the multi-GPU runs that check those releases cover single-part HBM
        // units only, so shared windows keep one part per HBM unit.
        const int32_t hbm_part_bytes = p.shared ? 0 : p.part_bytes;
        if ((rc = plan_gemm_operands(tasks, ntasks, tiles, ntiles, plan, why)) != PB2_SUCCESS) return rc;
        // Read groups as in HBM windows, except with priority lanes and one GEMM worker: such a window retires in the
        // oracle's priority order (tests/priority_order.py, DESIGN.md §6), and a group runs its members in its leader's
        // lane, one after the other, where the priority order may run a member of another lane, or a task one member
        // releases into a higher lane, in between.  An HBM window states that order for DAGs without groups only.
        if (p.queue_policy == 1 && p.nworkers_gemm == 1) plan.succ.assign(succ, succ + nsucc);
        else plan_read_groups(p, p.nworkers_gemm, succ, nsucc, tiles, ready, nready, plan);
        if ((rc = build_gemm2_units(p, plan.tasks.data(), ntasks, plan.succ.data(), ready, nready, p.gemm_mode == 0,
                                    p.shared ? p.next_rs_begin : nullptr, task_lane, tiles, hbm_part_bytes, plan, own, why)) != PB2_SUCCESS)
            return rc;
    }
    if (prio) build_lane_ring(plan, own);
    const int maxw = p.nworkers > p.nworkers_gemm ? p.nworkers : p.nworkers_gemm;
    uint32_t cap = 1024;
    while (cap < own.ring_slots + (uint32_t)maxw + 2u) cap <<= 1;   // every slot is used at most once per run
    plan.run.ring = cap;
    return PB2_SUCCESS;
}

}  // namespace pb2
