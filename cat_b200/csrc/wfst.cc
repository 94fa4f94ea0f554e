// Decoding-graph loader (wfst.h).  Host only.
#include "wfst.h"

#include <algorithm>
#include <cmath>

#include "den_graph.h"

namespace ccb {

bool LoadWfst(const char *path, WfstHost *out, std::string *err) {
    if (!path) { *err = "null path"; return false; }
    HostFst f;
    if (!ReadFstFile(path, &f, err, true)) return false;
    WfstHost &g = *out;
    g = WfstHost();
    const int S = f.num_states;
    const long A = (long)f.src.size();
    g.S = S;
    g.start = f.start;
    g.A = A;
    // layout: per state (the file lists arcs state by state), emitting arcs then epsilon arcs, each in file order
    g.arc_off.assign(S + 1, 0);
    g.eps_off.assign(S, 0);
    std::vector<int> n_emit(S, 0);
    for (long i = 0; i < A; ++i) {
        ++g.arc_off[f.src[i] + 1];
        if (f.label[i] >= 0) ++n_emit[f.src[i]];
    }
    for (int s = 0; s < S; ++s) {
        g.arc_off[s + 1] += g.arc_off[s];
        g.eps_off[s] = g.arc_off[s] + n_emit[s];
        g.max_out = std::max(g.max_out, n_emit[s]);
    }
    g.dst.resize(A); g.tok.resize(A); g.olabel.resize(A); g.fid.resize(A); g.src.resize(A); g.w.resize(A); g.lay.resize(A);
    std::vector<int> ce(S), cx(S);
    for (int s = 0; s < S; ++s) { ce[s] = g.arc_off[s]; cx[s] = g.eps_off[s]; }
    for (long i = 0; i < A; ++i) {
        const int s = f.src[i];
        const int j = f.label[i] >= 0 ? ce[s]++ : cx[s]++;
        g.dst[j] = f.dst[i];
        g.tok[j] = f.label[i];
        g.olabel[j] = f.olabel[i];
        g.fid[j] = (int)i;
        g.src[j] = s;
        g.w[j] = -f.logw[i];
        g.lay[i] = j;
        g.max_ilabel = std::max(g.max_ilabel, f.label[i] + 1);
        if (f.label[i] < 0) ++g.eps_arcs;
    }
    g.final_cost.resize(S);
    for (int s = 0; s < S; ++s) g.final_cost[s] = -f.final_logw[s];

    // epsilon levels by Kahn's algorithm over the epsilon subgraph: level = the longest epsilon path into the state
    std::vector<int> indeg(S, 0);
    for (int s = 0; s < S; ++s)
        for (int j = g.eps_off[s]; j < g.arc_off[s + 1]; ++j) ++indeg[g.dst[j]];
    g.level.assign(S, 0);
    std::vector<int> order;
    order.reserve(S);
    for (int s = 0; s < S; ++s)
        if (indeg[s] == 0) order.push_back(s);
    for (size_t k = 0; k < order.size(); ++k) {
        const int s = order[k];
        for (int j = g.eps_off[s]; j < g.arc_off[s + 1]; ++j) {
            const int d = g.dst[j];
            g.level[d] = std::max(g.level[d], g.level[s] + 1);
            if (--indeg[d] == 0) order.push_back(d);
        }
    }
    if ((int)order.size() != S) {
        // every state left has an epsilon predecessor that is left too: walking back through them must repeat a state,
        // and the first repeated state lies on a cycle
        std::vector<std::vector<int>> pred_left(S);
        for (int s = 0; s < S; ++s)
            if (indeg[s] > 0)
                for (int j = g.eps_off[s]; j < g.arc_off[s + 1]; ++j)
                    if (indeg[g.dst[j]] > 0) pred_left[g.dst[j]].push_back(s);
        int q = 0;
        while (indeg[q] == 0) ++q;
        std::vector<char> seen(S, 0);
        while (!seen[q]) { seen[q] = 1; q = pred_left[q][0]; }
        *err = std::string(path) + ": the epsilon arcs of the decoding graph form a cycle through state " + std::to_string(q) +
               "; the search needs an acyclic epsilon subgraph (remove the disambiguation-symbol loops, e.g. with "
               "`fstrmsymbols` on the disambiguation ids, only after determinization)";
        return false;
    }
    for (int s = 0; s < S; ++s) g.L = std::max(g.L, g.level[s]);
    // the largest epsilon closure: states reached through one or more epsilon arcs, by a search from every state that has
    // epsilon arcs (stamps instead of clearing a visited set)
    std::vector<int> stamp(S, -1), stack;
    for (int s = 0; s < S; ++s) {
        if (g.eps_off[s] == g.arc_off[s + 1]) continue;
        int n = 0;
        stack.assign(1, s);
        while (!stack.empty()) {
            const int q = stack.back();
            stack.pop_back();
            for (int j = g.eps_off[q]; j < g.arc_off[q + 1]; ++j) {
                const int d = g.dst[j];
                if (stamp[d] == s) continue;
                stamp[d] = s;
                ++n;
                stack.push_back(d);
            }
        }
        g.E = std::max(g.E, n);
    }
    return true;
}

}  // namespace ccb
