// Host-side den-graph loader and kernel plan (no CUDA in this header).
//
// Replaces the reference's loader src/ctc_crf/gpu_den/fst_read.cc:11-61 (OpenFst) and the CSR flattening
// in den_calculate.cu:309-355 with a native parser plus a plan laid out for the persistent kernels in
// den_kernels.cu.  See DESIGN.md "Data layout".
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace ccb {

// One arc as the kernels read it: 8 bytes, broadcast-loaded from shared memory two at a time (LDS.128).
//   peer : row of the gather table the arc reads: a state id (< S) or, in the forward pass, S + j for the
//          virtual row of pair j (the sum of the pair's two alphas, see DenPlan).
//   w    : arc weight in the LINEAR domain, exp(-tropical weight), always >= 0.  Arc segments are padded with
//          zero-weight arcs to whole QUADS of 4 arcs.  SIGN BITS of the last quad of a segment carry the event
//          (applied as |w| in the FMA): sign(w[3]) = "a segment ends here", sign(w[2]):sign(w[1]) = event code,
//          sign(w[0]) = "this row's label differs from the previous row of the same position in the chunk".
struct alignas(8) Arc {
    uint32_t peer;
    float w;
};
static constexpr int kQuad = 4;          // arcs per quad (segment padding granule)
static constexpr int kChunkArcPad = 16;  // every warp chunk's arc count is padded to a multiple of this
// event codes
static constexpr int kEvRow = 0;         // end of the row of an unpaired state
static constexpr int kEvRowPos0 = 1;     // end of the row of the first member of a pair
static constexpr int kEvRowPos1 = 2;     // end of the row of the second member of a pair
static constexpr int kEvPartial = 3;     // forward only: a PART of a high in-degree row; the last slot of the segment carries
                                         // the target row (weight 0) and the result is added to it atomically
static constexpr int kEvPairMerged = 3;  // forward only, plans WITHOUT high in-degree rows (same code as kEvPartial, which such plans never
                                         // contain): the segment ends BOTH rows of a pair.  Slots 0 .. n-2 are the in-arcs of the second
                                         // member, the LAST slot is the single in-arc of the first member (DenPlan::fwd_merged);
                                         // with own-row terms (DenPlan::own_rows) there is no such tail slot: all slots are the second member's
static constexpr int kHubInArcs = 384;   // rows with more in-arcs than this are split into parts of kPartArcs arcs that
static constexpr int kPartArcs = 191;    // any warp of the grid can own (real n-gram den graphs have such states)

// Den graph as stored in the file, in the view fst_read.cc:40-59 gives the kernels.
struct HostFst {
    int num_states = 0;
    int start = 0;
    std::vector<int> src, dst, label;   // label = ilabel-1
    std::vector<float> logw;            // -tropical
    std::vector<float> final_logw;      // -Final, -inf for non-final states
    std::vector<int> olabel;            // decoding graphs only (ReadFstFile decoding = true): the output label of every arc
};

// Returns false and fills err on failure (never exits, unlike den_calculate.cu:16-25,331-334).  decoding = false reads a den
// graph (epsilon input labels refused, olabels dropped); true reads a decoding graph (wfst.h): epsilon input labels are kept
// as label -1, olabels are kept, and const FSTs, symbol tables and aligned files are refused with the conversion to run.
bool ReadFstFile(const char *path, HostFst *out, std::string *err, bool decoding = false);

// Pass-specific half of the plan: a chunk-major stream of arc segments.  chunk_* cut the states (whole groups)
// into n_ctas*n_warps contiguous chunks of near-equal cost; CTA c owns chunks [c*n_warps, (c+1)*n_warps).
struct PassPlan {
    std::vector<Arc> arcs;              // chunk-major: segments as whole quads, chunk tails padded with unflagged zero quads
    std::vector<float> w1;              // backward only: second weight of every slot (see DenPlan::bwd)
    std::vector<int> chunk_state;       // [n_chunks+1] first state of each chunk
    std::vector<int> chunk_arc;         // [n_chunks+1] first arc of each chunk (multiples of kChunkArcPad)
    std::vector<int> chunk_pair;        // [n_chunks+1] first pair (virtual row) of each chunk
    std::vector<int> cta_labels;        // [n_ctas][4] = {min label of pos0 rows, #labels, min label of other rows, #labels}
    int real_arcs = 0;                  // arcs in this pass's stream (before padding)
    int max_tile_arcs = 0;              // max arcs owned by one CTA
    int max_tile_labels = 0;            // max rows of the per-CTA label accumulator (both ranges)
    int max_tile_rows = 0;              // max states owned by one CTA
};

struct DenPlan {
    int file_states = 0, file_arcs = 0;
    int num_states = 0;                 // S: states after the in-label split
    int num_pairs = 0;                  // P: paired states = 2P; virtual rows S..S+P-1 in the forward gather table
    int start = 0;                      // renumbered start state
    int num_labels = 0;                 // max label + 1
    int n_ctas = 0, n_warps = 0;
    int scale_exp = 56;                 // the kernels renormalise every column sum to ~2^scale_exp: 56, lowered when a state's
                                        // out-weight sum G is large so that alpha * beta <= 2^(2E+2) G^2 stays below 2^127
    std::vector<int> state_label;       // [S] the single label carried by every arc INTO the state
    std::vector<int> state_pos;         // [S] 0 = first member of a pair, 1 = second member or unpaired
    std::vector<float> final_lin;       // [S] exp(final_logw) (0 for non-final)
    std::vector<int> orig_state;        // [S] state id in the file
    std::vector<Arc> start_arcs;        // out-arcs of the start state (plain), for logZ recomputed from beta
    std::vector<int> hub_states;        // states whose forward row is accumulated from parts (rows zeroed before each frame)
    // fwd: one segment per state (its in-arcs; peers may be virtual pair rows), events kEvRow / kEvRowPos0 / kEvRowPos1;
    //      a high in-degree state has several kEvPartial segments instead (one in its own group, the others floating).
    //      fwd_merged (T-compose-LM graphs: the blank twin (h,B) of every pair has ONE in-arc, the pair's own virtual row):
    //      every pair is ONE segment, event kEvPairMerged -- the second member's in-arcs, then zero-weight padding, then the
    //      first member's arc in the last slot of the last quad.  28 instead of 28 + 4 padded slots per pair of a 24-successor
    //      LM and one row-end event instead of two: -12.5 % forward slots, forward pass 23.4 -> 20.5 ms at the headline size.
    //      The label-changed flag (sign of w[0] of the last quad) is the SECOND member's; all first members share one label.
    bool fwd_merged = false;
    // OWN-ROW terms (own_rows): arcs whose SOURCE row belongs to the destination's own group -- in a T-compose-LM graph the
    // blank arcs into (h,B), the token self loop of (h,L); in the backward pass the arcs from (h,B) / (h,L) to (h,B) / (h,L) --
    // name rows the same warp wrote one frame earlier.  They leave the gather streams: row q receives
    //     own[2q] * X(first row of its group) + own[2q+1] * X(second row of its group, or the row itself if unpaired)
    // on top of its gathered sum, X = the previous frame's alpha rows (forward) / the next frame's beta-hat rows (backward),
    // which the kernels fetch with two plain row loads per group, one group ahead of use.  Frame time follows the number of
    // slots a warp walks through its TMA ring, so this removes gathered slots from both passes.  All or nothing: only plans without hub rows in which every pair's first
    // member is left with NO gathered in-arc (then every pair is one merged forward segment without a tail slot).
    bool own_rows = false;
    std::vector<float> own_fwd, own_bwd;   // [2S + 4] (zero when !own_rows; padded so that a 4-float read at 2q stays inside)
    // bwd: one segment per GROUP (an unpaired state, or a pair p0,p1): every slot carries two weights, arcs[i].w for the
    //      group's first row and w1[i] for its second row (0 when the arc does not belong to that row), so the arcs the
    //      two members share are gathered once.  Event kEvRow = one-row group, kEvRowPos1 = two-row group; the
    //      label-changed flags of the two rows are sign(w[0]) and sign(w[1]) of the last quad.
    PassPlan fwd, bwd;
    // Plain in-arc CSR of the split graph in this renumbering, for the posterior sampler (den_sample.cu): the in-arcs of
    // state q are in_off[q] .. in_off[q+1]-1, each with its source state in_src and its LINEAR weight in_w.  Every arc once:
    // no pairs, no own-row coefficients, no padding, no event bits.
    std::vector<int> in_off, in_src;
    std::vector<float> in_w;
    // The same arcs as an out-arc CSR, for the prefix beam search (beam_search.cu): the out-arcs of state p are
    // out_off[p] .. out_off[p+1]-1, sorted by the label of their destination out_dst (then by out_dst), with LINEAR weights
    // out_w, so that the arc of p into a state of label c is found by binary search.
    std::vector<int> out_off, out_dst;
    std::vector<float> out_w;
};

// The condition under which a CTC prefix beam search over the plan's split graph is exact with two slots per prefix
// (DESIGN.md §7 "Prefix beam search"): no state has two out-arcs into states of one label, and every prefix reachable from
// the start state keeps ONE state in its blank slot and ONE in its token slot -- both slots step into the same state on a
// new token, the token slot repeats in place, the blank slot stays in place.  Breadth-first search over the signatures
// (blank-slot state, token-slot state) of the prefixes.  Returns false and names the states in *err when it does not hold.
bool CheckCtcShape(const DenPlan &plan, std::string *err);

// Build the plan:
//  1. split every state by the label of its incoming arcs so that each state has exactly one in-label
//     (a no-op for T-compose-LM graphs: build_ctc_topo.py:49-60 gives every arc into token state i the
//     ilabel i+1); this lets the kernels hoist the emission term out of the arc loop:
//         alpha_t(q) = y_{t-1}[lab(q)] * sum_p w_pq alpha_{t-1}(p)
//     and turns the per-arc atomic gradient of den_calculate.cu:219-223 into a per-state product
//         gamma_t[k] = sum_{q: lab(q)=k} alpha_{t+1}(q) beta_{t+1}(q) / Z.
//  2. PAIR states that feed the same destinations with bit-equal weights (in a T-compose-LM graph the blank and
//     label twins (h,B),(h,L) of an LM history h: ~all their out-arcs).  For a pair (p0,p1) with common
//     destinations C: the forward pass gathers ONE virtual row alpha(p0)+alpha(p1) per destination in C instead of
//     two rows; the backward pass sums the arcs into C once and reuses the partial sum for both members.  Exact
//     (sums are regrouped, nothing is approximated) and generic (pairs are found from the arc lists; an unpaired
//     state is a group of one).  Halves the gathers of a T-compose-LM graph.
//  3. order states group by group (pairs adjacent: p0 then p1), groups sorted by the label of their last member,
//     so a CTA tile spans few labels;
//  4. emit the forward (in-arc) and backward (out-arc) segment streams with linear-domain weights and cut them
//     into cost-balanced chunks for an n_ctas x n_warps persistent grid.
bool BuildDenPlan(const HostFst &fst, int n_ctas, int n_warps, DenPlan *plan, std::string *err);

}  // namespace ccb
