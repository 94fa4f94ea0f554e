// Host-side loader of a back-off n-gram LM in ARPA text, for token-level shallow fusion in the prefix beam search
// (beam_search.cu, DESIGN.md §7 "N-gram LM fusion").  No CUDA in this header.
#pragma once
#include <string>
#include <vector>

namespace ccb {

constexpr int kNgramMaxOrder = 10;

// The LM as the search walks it.  Words are the ARPA words some label names, plus <unk> (substituted with log10 p = -100
// when the file has none), </s> and <s> when the file lists them; word w is the unigram state 1 + w.
//   States: 0 is the root (the empty history), then every n-gram of order < n (after prefix closure: a listed n-gram's
//   missing prefixes are inserted with bow 0, and their arc carries probability NaN: "the back-off value", which the walk
//   computes by backing off after taking the arc's destination).
//   Arcs: each listed n-gram (h, w) of order >= 2 is an arc from state h, CSR over states, each state's arcs sorted by
//   word; its destination is the longest suffix of h.w that is a state.  The root's arcs are the dense root_p / root_dst.
//   back[s]: the longest proper suffix of s that is a state.  Values are ARPA log10, as parsed, in fp32.
// Scoring word w from state s: while s has no arc of w with a probability, add bow[s] and move to back[s]; at the root use
// root_p[w].  The next state is the destination of the first arc of w met (root_dst[w] if none).
struct NGramHost {
    int order = 0, V = 0, W = 0;
    long counts[kNgramMaxOrder] = {};   // n-grams per order as the \data\ section declares them
    bool unk_substituted = false;
    int bos = 0;                        // state after <s> (the root when the file lists no <s>)
    int eos = 0;                        // word id of </s> (<unk> when the file lists none)
    int bos_word = -1;                  // word id of <s>, -1 when the file lists none
    bool eos_listed = false;            // the file lists </s>
    std::vector<int> tok2word;          // [V]: -1 for the blank (token 0), <unk> for a label the LM does not list
    std::vector<float> root_p;          // [W]
    std::vector<int> root_dst;          // [W]
    std::vector<int> arc_off;           // [S + 1]
    std::vector<int> arc_word, arc_dst; // [A]
    std::vector<float> arc_p;           // [A]
    std::vector<float> bow;             // [S]
    std::vector<int> back;              // [S] (-1 for the root)
    int num_states() const { return (int)bow.size(); }
    long num_arcs() const { return (long)arc_word.size(); }
};

// Parse `path` for the token labels labels[0..V) (labels[0] is the blank and is never scored).  On failure returns false
// with *err naming the line.
bool LoadArpa(const char *path, const char *const *labels, int V, NGramHost *out, std::string *err);

}  // namespace ccb
