// Launch of the persistent den kernels: the variant that runs a pass and its dynamic shared memory, chosen on the host without
// a CUDA call (den_graph.cc).  Kernels carve with the strides and offsets below, and with the ring offsets in DenParams.
#pragma once
#include "den_graph.h"

#ifdef __CUDACC__
#define CCB_HD __host__ __device__
#else
#define CCB_HD
#endif

namespace ccb {

constexpr int kDenThreads = 512;   // 16 warps per CTA, one CTA per SM (the den plan is built for 16 warps per CTA)
// Backward arc bytes per CTA tile (12 per slot) above which a graph runs the large-graph tiers; only such graphs carry the
// streamed-arc copy of their backward quads, and their plans keep no own-row terms (den_graph.cc).
constexpr size_t kStreamTierArcBytes = 72 * 1024;
inline bool LargeGraphTiers(int bwd_max_tile_arcs) { return (size_t)bwd_max_tile_arcs * 12 > kStreamTierArcBytes; }

// Small-batch tier, per warp and stage: kSmallRows rows of 16 floats, an mbarrier, a 64-byte slot of streamed second weights
// (the slots of all warps follow all the mbarriers: SmallW1Off).
constexpr int kSmallLanes = 16, kSmallStages = 4, kSmallRows = 16;
constexpr uint32_t kSmallRingWarpBytes = kSmallStages * kSmallRows * kSmallLanes * 4, kSmallBarWarpBytes = kSmallStages * 8;
constexpr uint32_t kSmallW1WarpBytes = kSmallStages * 64;
// Streamed-arc tier, per warp: 2 stages of kStreamRows full-width rows, kArcStages batches of arc words, their mbarriers.
constexpr int kStreamRows = 16, kArcStages = 8;
CCB_HD constexpr uint32_t StreamRingWarpBytes(int U) { return 2u * kStreamRows * 32u * (uint32_t)U * 4u; }
constexpr uint32_t kStreamBarWarpBytes = 2 * 8, kArcBarWarpBytes = kArcStages * 8;
constexpr uint32_t kArcRingWarpBytes = kArcStages * (kStreamRows / kQuad) * 3 * 16;
// Gathers per batch of the register-gather kernels (two in flight per warp), fixed by the register budget at 512 threads.
CCB_HD constexpr int FwdBatch(int U) { return U == 4 ? 8 : 16; }
constexpr int kBwdBatch = 8;
// The arc tile follows the per-CTA bookkeeping at a 16-byte boundary.  Forward: column sums [Npad], row labels [tile_rows];
// backward: column sums [2][Npad], label accumulator [gacc_rows][Npad], row labels and final weights [tile_rows] each.
CCB_HD inline size_t FwdArcsOff(int Npad, int tile_rows) { return ((size_t)(Npad + tile_rows) * 4 + 15) & ~(size_t)15; }
CCB_HD inline size_t BwdArcsOff(int Npad, int gacc_rows, int tile_rows) {
    return ((((size_t)(2 + gacc_rows) * Npad + 2 * (size_t)tile_rows) * 4 + 15) & ~(size_t)15);
}
CCB_HD inline uint32_t SmallW1Off(uint32_t bar_off, int n_warps) { return bar_off + (uint32_t)n_warps * kSmallBarWarpBytes; }

struct DenPassShape { int max_tile_arcs = 0, max_tile_rows = 0, max_tile_labels = 0; };
// streamed_quads: the backward quads also exist in the streamed-arc form (DevicePass::tq); own_rows: DenPlan::own_rows
struct DenGraphShape { DenPassShape fwd, bwd; int n_hubs = 0, n_warps = 0; bool streamed_quads = false, own_rows = false; };
// test hooks CCB_ARCS_IN_GLOBAL, CCB_W1_IN_GLOBAL (force the large-graph tiers), CCB_NO_TMA (register gathers everywhere) and
// CCB_OWN_IN_L2 (own rows re-read from L2, not kept on chip)
struct DenHooks { bool arcs_in_global = false, w1_in_global = false, no_tma = false, own_in_l2 = false; };

// Arcs resident in shared memory or read from L2 with rows gathered into registers; backward only, arcs streamed through
// bulk-copy rings with rows staged by TMA; Npad = 16, arcs resident and 16-float rows staged by bulk copies.
enum DenTier { kTierShared, kTierGlobal, kTierStreamed, kTierSmall };
struct DenLaunch {
    int tier = kTierShared, lanes_per_row = 32, U = 1, batch = 0;   // U: utterances per lane; batch: gathers (rows) per batch
    bool w1_smem = false;   // backward: second weights resident with the arc tile (12 bytes per slot, else 8)
    int tile_rows = 0, gacc_rows = 0;
    // register tiers of a plan with own-row terms: the CTA tile's own rows of the last frame, [tile_rows][Npad] floats at
    // own_off, so that a warp reads back the rows it wrote itself from shared memory instead of L2
    bool own_smem = false;
    // dynamic shared memory in bytes from its base (0: a region the tier does not have)
    size_t arcs_off = 0, ring_off = 0, bar_off = 0, w1_off = 0, abar_off = 0, aring_off = 0, own_off = 0, total = 0;
};

// The launch of one pass at lane padding Npad with smem_optin bytes of shared memory per block; false, why, if none runs it.
bool ChooseDenLaunch(const DenGraphShape &g, int Npad, bool backward, int smem_optin, const DenHooks &hooks, DenLaunch *out,
                     std::string *why);
// both passes run the small-batch tier at Npad = 16: batches of <= 16 utterances are padded to 16 lanes (PadLanes)
bool SmallBatchOk(const DenGraphShape &g, int smem_optin, const DenHooks &hooks);
DenGraphShape ShapeOf(const DenPlan &plan, const DenHooks &hooks);

}  // namespace ccb
