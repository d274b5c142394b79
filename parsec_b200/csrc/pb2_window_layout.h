// pb2_window_layout.h -- what the window kernels and the host planner (pb2_window_plan.cpp) both read: ring entries,
// priority lanes, read-group words, GEMM units and the part rule.  Host/device neutral: it includes only the public
// engine header and standard headers, so the planner compiles without the CUDA toolkit.
#pragma once
#include <stdint.h>
#include "../../include/pb2_engine.h"

#ifdef __CUDACC__
#define PB2_HD __host__ __device__
#else
#define PB2_HD
#endif

namespace pb2 {

constexpr int32_t kEmpty = -1;

// Hot control words, one per 128-byte line so that atomics on them do not false-share.
struct alignas(128) Line { unsigned long long v; unsigned long long pad[15]; };

// Priority policy (queue_policy 1): PB2_PRIO_LANES FIFO lanes, lane 0 popped first.  pb2_window_create ranks the
// distinct priorities of the window's tasks, highest first; with at most PB2_PRIO_LANES of them a value's lane is its
// rank r (the reference's order exactly: higher priority first, FIFO among equals), otherwise floor(r * LANES / n).
// Each lane owns a contiguous segment of the ring as long as the entries its owners can ever push, so nothing wraps
// and head / tail are absolute ring indices.  avail counts the entries pushed and not yet claimed: a popper takes one
// from it before it takes a head ticket, so a ticket never runs past the entries that exist.
#define PB2_PRIO_LANES 16
struct Lanes {
    Line head[PB2_PRIO_LANES];        // next slot to pop
    Line tail[PB2_PRIO_LANES];        // next slot to push
    Line avail[PB2_PRIO_LANES];       // entries reserved by pushers and not claimed yet (may dip below 0 briefly)
    uint32_t begin[PB2_PRIO_LANES];   // first slot of each lane's segment
    uint32_t ninit[PB2_PRIO_LANES];   // initial ready entries at the start of each segment
};

#define PB2_GROUP_MAX 8     // members per read group (at most 15: the count is 4 bits of group[])
#define PB2_GROUP_FUSED 0x80000000u   // group[] of a producer that runs with its group as one unit
// pb2_task_t::flags of a window's device descriptors, set by the planner (the caller's flags keep bits 0..2): the body is
// a linked reader (PB2_LINK_READERS), whose results add up over parts and calls (store_result)
#define PB2_TASK_READER 0x80
// ... and a reader whose read group calls its group form (PB2_LINK_READER_GROUPS, run_linked_group_part)
#define PB2_TASK_READER_GROUP 0x40
// ... and a GEMM-worker body (PB2_LINK_GEMM_BODIES): in the linked GEMM kernels it gets the operand ring as scratch
#define PB2_TASK_GEMM_BODY 0x20

// A task whose tiles are large is executed as several PARTS (byte slices of its tiles) by different workers: one
// tile at HBM / NVLink speed needs the whole GPU (a 64-thread CTA keeps 4 KiB in flight; a 4 MiB tile is 1.3 us of
// the machine, not 1 ms of one CTA).  Parts per task (1..512) live in WinDev::nparts; ring entries of HBM windows
// are (part << 22) | task, so such a window holds at most 2^22 tasks when it has wide tasks.
#define PB2_MAX_PARTS 512
#define PB2_SLICE_WORDS (PB2_MAX_PARTS / 32)   // claim words per tile of sliced stage-in (stage_in_slices)
#define PB2_ENT_MAKE(task, part) ((int32_t)(((uint32_t)(part) << 22) | (uint32_t)(task)))
#define PB2_ENT_TASK(e)          ((int32_t)((uint32_t)(e) & 0x3FFFFFu))
#define PB2_ENT_PART(e)          ((int)((uint32_t)(e) >> 22))

// GEMM windows (pb2_gemm.cuh): the scheduling entities are units, each a chain of segments (member tasks).
struct GUnit {                  // 48 bytes, read-only
    int32_t seg_begin, seg_count;   // members, in chain order
    int32_t succ_begin, succ_count; // out-edges of all members (chain links removed): target unit ids
    int32_t dep_goal;               // in-edges from other units
    int32_t nparts;                 // ring entries: min(sub-tiles of C, kMaxParts) for GEMM units; for an HBM body
                                    // min(ceil(widest tile / part_bytes), kMaxParts) byte slices (1 in shared windows)
    int32_t tileC;                  // GEMM units: the C tile; -1 otherwise
    int32_t M, N, K;
    int32_t flags;                  // bit0 is_gemm, bit1 pushout C, bit2 a producer that runs with its read group
    int32_t pad;
};
struct GSeg { int32_t task, tileA, tileB, pad; };

namespace gemm {
constexpr int BM = 128, BN = 256;  // a C sub-tile: one part of a GEMM unit runs every nparts-th of them
constexpr int kMaxParts = 32;      // the part index travels in the 5-bit flow field of a ring entry
// a task of a GEMM-worker body runs as up to PB2_GEMM_BODY_MAX_PARTS parts (pb2_engine_set_gemm_body_parts)
static_assert(PB2_GEMM_BODY_MAX_PARTS == kMaxParts, "a GEMM-worker body's part index travels in a ring entry's part field");
}  // namespace gemm

// Application device bodies linked into HBM windows (pb2_engine_link_bodies).
PB2_HD inline bool is_linked_body(int body) { return body >= PB2_BODY_LINKED_0 && body <= PB2_BODY_LINKED_7; }

// part_bytes of engines and streams whose parameters leave it 0
constexpr int32_t kDefaultPartBytes = 256 * 1024;

// The parts a task runs as: min(ceil(widest tile / part_bytes), cap) byte slices; one for a NOP body or part_bytes <= 0.
// tile_bytes(id) is the byte count of tile id.  The device cuts the slices of a tile by the same rule (tile_slices_of).
template <class TileBytes>
static inline int task_parts(const pb2_task_t& t, TileBytes tile_bytes, int32_t part_bytes, int cap) {
    if (part_bytes <= 0 || t.body == PB2_BODY_NOP) return 1;
    uint32_t big = 0;
    for (int f = 0; f < t.nb_flows; ++f)
        if (t.tile[f] >= 0 && tile_bytes(t.tile[f]) > big) big = tile_bytes(t.tile[f]);
    const uint32_t np = (big + (uint32_t)part_bytes - 1) / (uint32_t)part_bytes;
    return np < 1 ? 1 : (np > (uint32_t)cap ? cap : (int)np);
}

// The stage-in slice size of HBM windows and streams: the smaller of stage_slice_bytes and part_bytes among those that
// are positive, so a tile is never staged in coarser slices than wide tasks are cut into; part_bytes when neither is.
static inline int32_t stage_slice(int32_t stage_slice_bytes, int32_t part_bytes) {
    return (stage_slice_bytes > 0 && (part_bytes <= 0 || stage_slice_bytes < part_bytes)) ? stage_slice_bytes : part_bytes;
}

}  // namespace pb2

#undef PB2_HD
