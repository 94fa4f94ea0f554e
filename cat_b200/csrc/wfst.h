// Host-side decoding graph (TLG) for the frame-synchronous Viterbi beam search (wfst_decode.cu, DESIGN.md §7 "TLG
// decoding").  No CUDA in this header.
#pragma once
#include <string>
#include <vector>

namespace ccb {

// An OpenFst vector/standard decoding graph in CAT's conventions: ilabel = token + 1 (blank = token 0), ilabel 0 = epsilon,
// olabel = word id (0: no word), tropical weights.  Arcs are laid out per state, the state's emitting arcs first (in file
// order) and its epsilon arcs after (in file order): the arcs of state s are arc_off[s] .. arc_off[s+1]-1, the emitting
// ones end at eps_off[s].  fid is an arc's position in file order (the search's tie-break); lay inverts it.
struct WfstHost {
    int S = 0, start = 0;
    long A = 0, eps_arcs = 0;
    std::vector<int> arc_off, eps_off;          // [S + 1], [S]
    std::vector<int> dst, tok, olabel, fid, src;  // [A] in layout order; tok = ilabel - 1 (-1: epsilon)
    std::vector<float> w;                       // [A] tropical cost
    std::vector<int> lay;                       // [A] layout position of file arc i
    std::vector<float> final_cost;              // [S] tropical, +inf for non-final states
    std::vector<int> level;                     // [S] the longest epsilon path into the state
    int L = 0;             // the longest epsilon path
    int E = 0;             // the largest epsilon closure: the most states one state reaches through one or more epsilon arcs
    int max_out = 0;       // the largest emitting out-degree
    int max_ilabel = 0;    // the largest ilabel (the logits need at least this many labels)
};

// Read and check a decoding graph.  The epsilon subgraph must be acyclic (a cycle is refused, naming a state on it); const
// FSTs, embedded symbol tables and aligned files are refused with the conversion to run (den_graph.h ReadFstFile).
bool LoadWfst(const char *path, WfstHost *out, std::string *err);

}  // namespace ccb
