// Host-side den-graph loader, kernel plan and kernel launch decision.  See den_graph.h and den_launch.h.
#include "den_graph.h"
#include "den_launch.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <numeric>
#include <unordered_set>

namespace ccb {

namespace {

struct ByteReader {
    const unsigned char *p;
    size_t n, off = 0;
    bool ok = true;
    template <typename T> T get() {
        T v{};
        if (off + sizeof(T) > n) { ok = false; return v; }
        memcpy(&v, p + off, sizeof(T));
        off += sizeof(T);
        return v;
    }
    std::string str() {
        int32_t len = get<int32_t>();
        if (!ok || len < 0 || off + (size_t)len > n) { ok = false; return {}; }
        std::string s((const char *)p + off, (size_t)len);
        off += (size_t)len;
        return s;
    }
};

}  // namespace

// OpenFst binary container, "vector" fst of "standard" (tropical) arcs.  Layout: SURVEY.md 8c.
// Semantics: fst_read.cc:40-59 (weight negated, ilabel shifted by one, -inf for Zero finals).
// decoding: a decoding graph (wfst.h) -- olabels are kept and ilabel 0 (epsilon, label -1) is accepted; the refusals name
// the conversion that makes a file readable.
bool ReadFstFile(const char *path, HostFst *out, std::string *err, bool decoding) {
    const std::string what = decoding ? "decoding graph" : "den graph";
    FILE *f = fopen(path, "rb");
    if (!f) { *err = "cannot open " + what + ": " + path; return false; }
    fseek(f, 0, SEEK_END);
    long sz = ftell(f);
    fseek(f, 0, SEEK_SET);
    std::vector<unsigned char> buf((size_t)std::max(sz, 0L));
    size_t got = sz > 0 ? fread(buf.data(), 1, (size_t)sz, f) : 0;
    fclose(f);
    if ((long)got != sz) { *err = std::string("short read: ") + path; return false; }

    ByteReader r{buf.data(), buf.size()};
    if ((uint32_t)r.get<int32_t>() != 0x7EB2FDD6u) { *err = std::string("not an OpenFst binary file: ") + path; return false; }
    std::string fst_type = r.str(), arc_type = r.str();
    if (decoding && r.ok && fst_type == "const") {
        *err = what + " " + path + " is a const FST; convert it with `fstconvert --fst_type=vector`";
        return false;
    }
    if (!r.ok || fst_type != "vector" || arc_type != "standard") {
        *err = "unsupported fst/arc type '" + fst_type + "'/'" + arc_type + "' (need vector/standard)";
        return false;
    }
    const int32_t version = r.get<int32_t>();
    const int32_t flags = r.get<int32_t>();
    if (r.ok && version != 2) { *err = "unsupported VectorFst file version " + std::to_string(version) + " (need 2)"; return false; }
    if (flags & 0x3) {
        *err = decoding ? what + " carries embedded symbol tables; strip them with `fstsymbols --clear_isymbols --clear_osymbols`"
                        : "den graph carries embedded symbol tables; strip them (fstsymbols --clear_*)";
        return false;
    }
    if (flags & 0x4) {
        *err = decoding ? what + " was written with aligned fields; rewrite it with `fstconvert --fst_align=false`"
                        : "den graph was written with aligned fields (FstHeader::IS_ALIGNED); rewrite it with --fst_align=false";
        return false;
    }
    (void)r.get<uint64_t>();  // properties
    int64_t start = r.get<int64_t>();
    int64_t ns = r.get<int64_t>();
    (void)r.get<int64_t>();   // header arc count: 0 in files written by fstcompile pipelines, not trusted
    if (!r.ok || ns <= 0 || ns > (int64_t)0x7fffffff || start < 0 || start >= ns) {
        *err = "corrupt " + what + " header";
        return false;
    }
    out->num_states = (int)ns;
    out->start = (int)start;
    out->final_logw.assign((size_t)ns, -std::numeric_limits<float>::infinity());
    out->src.clear(); out->dst.clear(); out->label.clear(); out->logw.clear(); out->olabel.clear();
    for (int64_t s = 0; s < ns; ++s) {
        float fin = r.get<float>();
        int64_t na = r.get<int64_t>();
        if (!r.ok || na < 0 || r.off + (size_t)na * 16 > r.n) { *err = "truncated " + what; return false; }
        if (!std::isinf(fin)) out->final_logw[(size_t)s] = -fin;
        for (int64_t a = 0; a < na; ++a) {
            int32_t il = r.get<int32_t>();
            const int32_t ol = r.get<int32_t>();
            float w = r.get<float>();
            int32_t nx = r.get<int32_t>();
            if (!decoding && (nx < 0 || nx >= ns || il < 1)) { *err = "den graph arc out of range (epsilon input labels are not allowed)"; return false; }
            if (decoding && (nx < 0 || nx >= ns || il < 0 || ol < 0)) {
                *err = what + " arc " + std::to_string(out->src.size()) + " out of range (state " + std::to_string(s) + ")";
                return false;
            }
            out->src.push_back((int)s);
            out->dst.push_back(nx);
            out->label.push_back(il - 1);
            out->logw.push_back(-w);
            if (decoding) out->olabel.push_back(ol);
        }
    }
    if (r.off != r.n) { *err = "trailing bytes in " + what; return false; }
    if (out->src.size() > (size_t)0x3fffffff) { *err = what + " too large"; return false; }
    return true;
}

namespace {

inline uint32_t Bits(float w) { uint32_t b; memcpy(&b, &w, 4); return b; }
inline float WithSign(float w) { uint32_t b = Bits(w) | 0x80000000u; float r; memcpy(&r, &b, 4); return r; }

struct Segment {
    std::vector<Arc> arcs;
    std::vector<float> w1;   // backward group segments only (same length as arcs)
    int event = kEvRow;
    int rows = 1;            // rows that end with this segment (0 for kEvCommon, 2 for a backward pair group / a merged forward pair)
    bool merged = false;     // forward kEvPairMerged: arcs = the second member's in-arcs [+ (last) the first member's single arc]
    bool tail = false;       // ... whether that tail arc is there (no own-row terms) or not
};
struct Group {
    std::vector<Segment> segs;
    int first_state = 0, rows = 0, pairs = 0;
};

// Cut groups into n_chunks contiguous chunks of near-equal cost and emit the chunk-major padded arc stream.
// Emit the chunk-major padded arc stream of one pass for the given chunk boundaries (chunk c = groups
// [chunk_group[c], chunk_group[c+1])).
void Layout(const std::vector<Group> &groups, int S, const std::vector<int> &state_label, const std::vector<int> &state_pos,
            int n_ctas, int n_warps, const std::vector<int> &chunk_group, bool emit_w1, PassPlan *pp) {
    const int G = (int)groups.size();
    const int n_chunks = n_ctas * n_warps;
    auto quads = [](const Segment &sg) { return std::max<int64_t>(1, ((int64_t)sg.arcs.size() + kQuad - 1) / kQuad); };
    pp->real_arcs = 0;
    for (int g = 0; g < G; ++g)
        for (auto &sg : groups[(size_t)g].segs) pp->real_arcs += (int)sg.arcs.size();

    pp->arcs.clear();
    pp->w1.clear();
    pp->chunk_state.assign((size_t)n_chunks + 1, S);
    pp->chunk_arc.assign((size_t)n_chunks + 1, 0);
    pp->chunk_pair.assign((size_t)n_chunks + 1, 0);
    int pairs_seen = 0;
    uint32_t last_peer = 0;
    for (int c = 0; c < n_chunks; ++c) {
        pp->chunk_arc[c] = (int)pp->arcs.size();
        pp->chunk_pair[c] = pairs_seen;
        pp->chunk_state[c] = chunk_group[c] < G ? groups[(size_t)chunk_group[c]].first_state : S;
        int prev_label[2] = {-1, -1};   // last label seen in this chunk per row position (-1: none yet)
        for (int g = chunk_group[c]; g < chunk_group[c + 1]; ++g) {
            const Group &gr = groups[(size_t)g];
            pairs_seen += gr.pairs;
            int row = gr.first_state;
            for (auto &sg : gr.segs) {
                // "label changed" flags: the row's label differs from the previous row of its position in this chunk;
                // the kernels then skip the label lookup / emission refresh on the common path.
                // one-row segments: sign(w[0]); two-row (backward pair) segments: sign(w[0]) for p0, sign(w[1]) for p1.
                bool chg0 = false, chg1 = false;
                if (sg.merged) {   // one flag: the SECOND member's label (first members all carry one label, checked by the builder)
                    prev_label[0] = state_label[(size_t)row];
                    chg0 = state_label[(size_t)row + 1] != prev_label[1];
                    prev_label[1] = state_label[(size_t)row + 1];
                } else if (sg.rows == 1 && sg.event != kEvPartial) {   // (partial rows bypass the kernels' emission cache)
                    const int k = sg.event == kEvRowPos0 ? 0 : 1;
                    chg0 = state_label[(size_t)row] != prev_label[k];
                    prev_label[k] = state_label[(size_t)row];
                } else if (sg.rows == 2) {
                    chg0 = state_label[(size_t)row] != prev_label[0];
                    prev_label[0] = state_label[(size_t)row];
                    chg1 = state_label[(size_t)row + 1] != prev_label[1];
                    prev_label[1] = state_label[(size_t)row + 1];
                }
                row += sg.rows;
                const size_t padded = (size_t)quads(sg) * kQuad;
                // Padding arcs carry weight 0 but are still gathered: point them at a row this warp reads anyway.
                // Pointing them all at one fixed row makes every warp of the grid hammer a single L2 line
                // (measured: 2x frame time from that hot spot alone).
                const uint32_t pad_peer = sg.arcs.empty() ? (uint32_t)gr.first_state : sg.arcs.back().peer;
                const bool dual = !sg.merged && (!sg.w1.empty() || sg.rows == 2);
                const size_t n_lead = sg.tail ? sg.arcs.size() - 1 : sg.arcs.size();   // merged with a tail: the last arc sits in the last slot
                const uint32_t pad_peer_m = sg.tail ? (n_lead ? sg.arcs[n_lead - 1].peer : sg.arcs.back().peer) : pad_peer;
                for (size_t i = 0; i < padded; ++i) {
                    Arc a = i < n_lead ? sg.arcs[i] : Arc{pad_peer_m, 0.f};
                    if (sg.tail && i + 1 == padded) a = sg.arcs.back();
                    if (i + 1 == padded) a.w = WithSign(a.w);
                    if (i + 2 == padded && (sg.event & 2)) a.w = WithSign(a.w);
                    if (dual) {
                        if (i + 3 == padded && chg1) a.w = WithSign(a.w);
                    } else {
                        if (i + 3 == padded && (sg.event & 1)) a.w = WithSign(a.w);
                    }
                    if (i + 4 == padded && chg0) a.w = WithSign(a.w);
                    pp->arcs.push_back(a);
                    if (emit_w1) pp->w1.push_back(i < sg.w1.size() ? sg.w1[i] : 0.f);
                }
                last_peer = pad_peer;
            }
        }
        while (pp->arcs.size() % kChunkArcPad) { pp->arcs.push_back(Arc{last_peer, 0.f}); if (emit_w1) pp->w1.push_back(0.f); }
    }
    pp->chunk_arc[n_chunks] = (int)pp->arcs.size();
    pp->chunk_pair[n_chunks] = pairs_seen;
    pp->chunk_state[n_chunks] = S;
    for (int c = n_chunks - 1; c >= 0; --c)   // empty trailing chunks start where the next one does
        if (chunk_group[c] == chunk_group[c + 1]) pp->chunk_state[c] = pp->chunk_state[c + 1];

    pp->max_tile_arcs = 0;
    pp->max_tile_labels = 1;
    pp->max_tile_rows = 1;
    pp->cta_labels.assign((size_t)n_ctas * 4, 0);
    for (int c = 0; c < n_ctas; ++c) {
        int a0 = pp->chunk_arc[(size_t)c * n_warps], a1 = pp->chunk_arc[(size_t)(c + 1) * n_warps];
        pp->max_tile_arcs = std::max(pp->max_tile_arcs, a1 - a0);
        int s0 = pp->chunk_state[(size_t)c * n_warps], s1 = pp->chunk_state[(size_t)(c + 1) * n_warps];
        pp->max_tile_rows = std::max(pp->max_tile_rows, s1 - s0);
        int lo[2] = {1 << 30, 1 << 30}, hi[2] = {-1, -1};
        for (int q = s0; q < s1; ++q) {
            const int k = state_pos[(size_t)q] ? 1 : 0;
            lo[k] = std::min(lo[k], state_label[(size_t)q]);
            hi[k] = std::max(hi[k], state_label[(size_t)q]);
        }
        int *cl = &pp->cta_labels[(size_t)c * 4];
        cl[0] = hi[0] >= 0 ? lo[0] : 0; cl[1] = hi[0] >= 0 ? hi[0] - lo[0] + 1 : 0;
        cl[2] = hi[1] >= 0 ? lo[1] : 0; cl[3] = hi[1] >= 0 ? hi[1] - lo[1] + 1 : 0;
        pp->max_tile_labels = std::max(pp->max_tile_labels, cl[1] + cl[3]);
    }
}

}  // namespace

static bool BuildDenPlanImpl(const HostFst &fst, int n_ctas, int n_warps, bool allow_own, DenPlan *plan, std::string *err);

bool BuildDenPlan(const HostFst &fst, int n_ctas, int n_warps, DenPlan *plan, std::string *err) {
    if (!BuildDenPlanImpl(fst, n_ctas, n_warps, true, plan, err)) return false;
    // Own-row terms are for graphs that run the main tier.  On the large-graph tiers (LargeGraphTiers: register gathers forwards,
    // streamed arcs backwards) the extra row loads and registers cost more than the dropped padding returns (5.1 M-arc
    // graph, N=128, T=2000: 615 ms per step with own-row terms against 575 ms without): build such a graph without them.
    if (plan->own_rows && LargeGraphTiers(plan->bwd.max_tile_arcs)) {
        *plan = DenPlan();
        return BuildDenPlanImpl(fst, n_ctas, n_warps, false, plan, err);
    }
    return true;
}

static bool BuildDenPlanImpl(const HostFst &fst, int n_ctas, int n_warps, bool allow_own, DenPlan *plan, std::string *err) {
    const int S0 = fst.num_states;
    const size_t A0 = fst.src.size();
    if (n_ctas < 1 || n_warps < 1) { *err = "bad grid for den plan"; return false; }

    // 1. distinct in-labels per file state; split states ("sid" = id after the split, sorted by label)
    std::vector<std::vector<int>> in_labels((size_t)S0);
    for (size_t a = 0; a < A0; ++a) in_labels[(size_t)fst.dst[a]].push_back(fst.label[a]);
    size_t S = 0;
    int max_label = 0;
    for (int q = 0; q < S0; ++q) {
        auto &v = in_labels[(size_t)q];
        std::sort(v.begin(), v.end());
        v.erase(std::unique(v.begin(), v.end()), v.end());
        if (v.empty()) v.push_back(0);  // no in-arcs (e.g. the start state): the label is never used
        S += v.size();
        max_label = std::max(max_label, v.back());
    }
    size_t A = 0;
    for (size_t a = 0; a < A0; ++a) A += in_labels[(size_t)fst.src[a]].size();
    if (S > (size_t)0x3fffffff || A > (size_t)0x3fffffff) {
        *err = "den graph too large after in-label state split (S=" + std::to_string(S) + ", A=" + std::to_string(A) + ")";
        return false;
    }
    struct Copy { int label, orig; };
    std::vector<Copy> copies;
    copies.reserve(S);
    for (int q = 0; q < S0; ++q) for (int k : in_labels[(size_t)q]) copies.push_back(Copy{k, q});
    std::stable_sort(copies.begin(), copies.end(), [](const Copy &a, const Copy &b) { return a.label < b.label; });
    std::vector<std::vector<int>> sid_of((size_t)S0);
    for (int q = 0; q < S0; ++q) sid_of[(size_t)q].assign(in_labels[(size_t)q].size(), -1);
    std::vector<int> sid_label(S), sid_orig(S);
    for (size_t i = 0; i < S; ++i) {
        const Copy &c = copies[i];
        auto &labs = in_labels[(size_t)c.orig];
        size_t j = (size_t)(std::lower_bound(labs.begin(), labs.end(), c.label) - labs.begin());
        sid_of[(size_t)c.orig][j] = (int)i;
        sid_label[i] = c.label;
        sid_orig[i] = c.orig;
    }
    struct SArc { int peer; float w; };
    std::vector<std::vector<SArc>> in_s(S), out_s(S);   // by sid
    for (size_t a = 0; a < A0; ++a) {
        const int p = fst.src[a], q = fst.dst[a];
        auto &labs = in_labels[(size_t)q];
        size_t j = (size_t)(std::lower_bound(labs.begin(), labs.end(), fst.label[a]) - labs.begin());
        const int qs = sid_of[(size_t)q][j];
        const float w = std::exp(fst.logw[a]);
        if (!(w >= 0.f) || std::isinf(w)) { *err = "den graph arc weight is not a finite probability-like value"; return false; }
        for (int ps : sid_of[(size_t)p]) {
            in_s[(size_t)qs].push_back(SArc{ps, w});
            out_s[(size_t)ps].push_back(SArc{qs, w});
        }
    }

    // hubs: states whose in-arc row is too long for one warp
    std::vector<char> is_hub(S, 0);
    {
        const char *e = getenv("CCB_HUB_IN_ARCS");   // test hook
        const size_t hub_thr = e ? (size_t)atoi(e) : (size_t)kHubInArcs;
        for (size_t q = 0; q < S; ++q) is_hub[q] = in_s[q].size() > hub_thr;
    }
    int part_arcs = kPartArcs;
    {
        const char *e = getenv("CCB_PART_ARCS");     // test hook; must leave the last slot of a quad for the target
        if (e && atoi(e) >= 3) part_arcs = atoi(e) / kQuad * kQuad + kQuad - 1;
    }

    // 2. pair detection: two sources that enter a destination with bit-equal weights, counted over destinations
    std::vector<int> partner(S, -1);
    {
        std::vector<std::pair<uint64_t, int>> keys;   // (p1<<32|p2) occurrences
        std::vector<uint64_t> occ;
        std::vector<std::pair<uint32_t, int>> tmp;
        for (size_t q = 0; q < S; ++q) {
            tmp.clear();
            for (auto &a : in_s[q]) tmp.emplace_back(Bits(a.w), a.peer);
            std::sort(tmp.begin(), tmp.end());
            for (size_t i = 0; i < tmp.size();) {
                size_t j = i;
                while (j < tmp.size() && tmp[j].first == tmp[i].first) ++j;
                if (j - i == 2 && tmp[i].second != tmp[i + 1].second)
                    occ.push_back(((uint64_t)(uint32_t)tmp[i].second << 32) | (uint32_t)tmp[i + 1].second);
                i = j;
            }
        }
        std::sort(occ.begin(), occ.end());
        struct Cand { int count, p1, p2; };
        std::vector<Cand> cands;
        for (size_t i = 0; i < occ.size();) {
            size_t j = i;
            while (j < occ.size() && occ[j] == occ[i]) ++j;
            if (j - i >= 2) cands.push_back(Cand{(int)(j - i), (int)(occ[i] >> 32), (int)(occ[i] & 0xffffffffu)});
            i = j;
        }
        std::sort(cands.begin(), cands.end(), [](const Cand &a, const Cand &b) {
            return a.count != b.count ? a.count > b.count : (a.p1 != b.p1 ? a.p1 < b.p1 : a.p2 < b.p2);
        });
        const char *nopair = getenv("CCB_NO_PAIRS");
        if (!(nopair && nopair[0] == '1'))
            for (auto &c : cands) {
                if (is_hub[(size_t)c.p1] || is_hub[(size_t)c.p2]) continue;   // hub rows are accumulated from parts
                if (partner[(size_t)c.p1] < 0 && partner[(size_t)c.p2] < 0) { partner[(size_t)c.p1] = c.p2; partner[(size_t)c.p2] = c.p1; }
            }
    }

    // 3. groups and final state order ("fid")
    struct GroupKey { int lab1, lab0, s0, s1, part; };   // s0 = pos0 sid or -1, s1 = pos1 sid; part > 0: floating part of hub s1
    std::vector<GroupKey> gk;
    for (size_t s = 0; s < S; ++s) {
        const int o = partner[s];
        if (o < 0) {
            gk.push_back(GroupKey{sid_label[s], -1, -1, (int)s, 0});
            if (is_hub[s]) {
                const int parts = (int)((in_s[s].size() + part_arcs - 1) / part_arcs);
                for (int j = 1; j < parts; ++j) gk.push_back(GroupKey{sid_label[s], -1, -1, (int)s, j});
            }
            continue;
        }
        if ((int)s > o) continue;   // handle each pair once
        int a = (int)s, b = o;      // pos0 = smaller label (ties: smaller sid)
        if (sid_label[(size_t)b] < sid_label[(size_t)a]) std::swap(a, b);
        gk.push_back(GroupKey{sid_label[(size_t)b], sid_label[(size_t)a], a, b, 0});
    }
    std::sort(gk.begin(), gk.end(), [](const GroupKey &x, const GroupKey &y) {
        if (x.lab1 != y.lab1) return x.lab1 < y.lab1;
        if (x.lab0 != y.lab0) return x.lab0 < y.lab0;
        if (x.s1 != y.s1) return x.s1 < y.s1;
        return x.part < y.part;
    });
    std::vector<int> fid(S, -1), pair_of(S, -1);
    std::vector<Group> fgroups, bgroups;
    auto by_peer = [](const Arc &a, const Arc &b) { return a.peer < b.peer; };
    struct Ent { int pair; uint32_t wb; int member; int peer_fid; float w; };
    std::vector<Ent> ents;
    struct OEnt { int q; uint32_t wb; float w; };
    std::vector<OEnt> l0, l1;

    // (re)number the states for a given group order and build both passes' segments
    auto build = [&](const std::vector<GroupKey> &order) {
        plan->state_label.assign(S, 0); plan->state_pos.assign(S, 1); plan->orig_state.assign(S, 0); plan->final_lin.assign(S, 0.f);
        int next = 0, n_pairs = 0;
        for (auto &g : order) {
            if (g.part > 0) continue;   // floating part of a hub row: no state of its own
            if (g.s0 >= 0) { fid[(size_t)g.s0] = next++; pair_of[(size_t)g.s0] = n_pairs; pair_of[(size_t)g.s1] = n_pairs; }
            fid[(size_t)g.s1] = next++;
            if (g.s0 >= 0) ++n_pairs;
        }
        plan->hub_states.clear();
        for (size_t s = 0; s < S; ++s) if (is_hub[s]) plan->hub_states.push_back(fid[s]);
        for (size_t s = 0; s < S; ++s) {
            const int f = fid[s];
            plan->state_label[(size_t)f] = sid_label[s];
            plan->orig_state[(size_t)f] = sid_orig[s];
            const float fw = fst.final_logw[(size_t)sid_orig[s]];
            plan->final_lin[(size_t)f] = std::isinf(fw) ? 0.f : std::exp(fw);
        }
        for (auto &g : order) if (g.s0 >= 0) plan->state_pos[(size_t)fid[(size_t)g.s0]] = 0;
        plan->num_pairs = n_pairs;
        plan->start = fid[(size_t)sid_of[(size_t)fst.start][0]];   // all start mass on one copy (copies share out-arcs)
        plan->start_arcs.clear();
        for (auto &a : out_s[(size_t)sid_of[(size_t)fst.start][0]]) plan->start_arcs.push_back(Arc{(uint32_t)fid[(size_t)a.peer], a.w});

        // forward rows: a pair's two arcs with equal weight become one arc to the pair's virtual row S + j
        auto forward_row = [&](int s, std::vector<Arc> *row) {
            ents.clear();
            for (auto &a : in_s[(size_t)s]) {
                const int pj = pair_of[(size_t)a.peer];
                const int member = pj >= 0 ? plan->state_pos[(size_t)fid[(size_t)a.peer]] : 0;
                ents.push_back(Ent{pj, Bits(a.w), member, fid[(size_t)a.peer], a.w});
            }
            std::sort(ents.begin(), ents.end(), [](const Ent &x, const Ent &y) {
                if (x.pair != y.pair) return x.pair < y.pair;
                if (x.wb != y.wb) return x.wb < y.wb;
                return x.member < y.member;
            });
            row->clear();
            for (size_t i = 0; i < ents.size();) {
                if (ents[i].pair < 0) { row->push_back(Arc{(uint32_t)ents[i].peer_fid, ents[i].w}); ++i; continue; }
                size_t j = i;
                int n0 = 0, n1 = 0;
                while (j < ents.size() && ents[j].pair == ents[i].pair && ents[j].wb == ents[i].wb) { (ents[j].member ? n1 : n0)++; ++j; }
                const int merged = std::min(n0, n1);
                for (int k = 0; k < merged; ++k) row->push_back(Arc{(uint32_t)(S + (size_t)ents[i].pair), ents[i].w});
                // leftovers keep their own rows: member-0 entries come first in [i, j)
                for (int k = merged; k < n0; ++k) row->push_back(Arc{(uint32_t)ents[i + (size_t)k].peer_fid, ents[i].w});
                for (int k = merged; k < n1; ++k) row->push_back(Arc{(uint32_t)ents[i + (size_t)n0 + (size_t)k].peer_fid, ents[i].w});
                i = j;
            }
            std::sort(row->begin(), row->end(), by_peer);
        };
        auto out_list = [&](int s, std::vector<OEnt> *l) {
            l->clear();
            for (auto &a : out_s[(size_t)s]) l->push_back(OEnt{fid[(size_t)a.peer], Bits(a.w), a.w});
            std::sort(l->begin(), l->end(), [](const OEnt &x, const OEnt &y) { return x.q != y.q ? x.q < y.q : x.wb < y.wb; });
        };
        // own-row terms (den_graph.h DenPlan::own_rows): move the arcs of `row` (forward row of sid s, group s0|s1) whose source
        // is one of the group's own rows -- real rows or the pair's virtual row -- into the coefficients; likewise backward
        bool own = false;
        auto extract_own_fwd = [&](int s, int s0, int s1, std::vector<Arc> *row, bool commit) {
            const int f = fid[(size_t)s];
            const uint32_t f0 = s0 >= 0 ? (uint32_t)fid[(size_t)s0] : 0xffffffffu, f1 = (uint32_t)fid[(size_t)s1];
            const uint32_t vr = s0 >= 0 ? (uint32_t)(S + (size_t)pair_of[(size_t)s0]) : 0xffffffffu;
            size_t k = 0;
            for (auto &a : *row) {
                float c0 = 0.f, c1 = 0.f;
                if (a.peer == f0) c0 = a.w;
                else if (a.peer == f1) c1 = a.w;
                else if (a.peer == vr) { c0 = a.w; c1 = a.w; }
                else { (*row)[k++] = a; continue; }
                if (commit) { plan->own_fwd[2 * (size_t)f] += c0; plan->own_fwd[2 * (size_t)f + 1] += c1; }
            }
            row->resize(k);
        };
        auto extract_own_bwd = [&](int s, int s0, int s1, std::vector<OEnt> *l) {
            const int f = fid[(size_t)s];
            const int f0 = s0 >= 0 ? fid[(size_t)s0] : -1, f1 = fid[(size_t)s1];
            size_t k = 0;
            for (auto &e : *l) {
                if (e.q == f0) plan->own_bwd[2 * (size_t)f] += e.w;
                else if (e.q == f1) plan->own_bwd[2 * (size_t)f + 1] += e.w;
                else (*l)[k++] = e;
            }
            l->resize(k);
        };
        fgroups.clear(); bgroups.clear();
        fgroups.reserve(order.size()); bgroups.reserve(order.size());
        std::vector<Arc> hub_row;
        // merged forward pairs (den_graph.h DenPlan::fwd_merged): all or nothing -- no hub rows anywhere, every first member
        // has exactly one in-arc, all first members carry the same label (the kernels refresh that emission once per frame)
        bool merge = plan->hub_states.empty() && plan->num_pairs > 0;
        {
            const char *e = getenv("CCB_NO_MERGE");   // test hook / A-B switch
            if (e && e[0] == '1') merge = false;
            int lab0 = -1;
            std::vector<Arc> probe;
            for (auto &g : order) {
                if (!merge) break;
                if (g.part > 0) { merge = false; break; }
                if (g.s0 < 0) continue;
                forward_row(g.s0, &probe);
                if (probe.size() != 1 || !(probe[0].w > 0.f)) merge = false;
                if (lab0 < 0) lab0 = g.lab0; else if (g.lab0 != lab0) merge = false;
            }
        }
        // own-row terms: all or nothing -- every pair's first member must be left without a gathered in-arc
        {
            const char *e1 = getenv("CCB_NO_OWN"), *e2 = getenv("CCB_NO_MERGE");   // test hooks / A-B switches
            own = allow_own && plan->hub_states.empty() && !(e1 && e1[0] == '1') && !(e2 && e2[0] == '1');
        }
        {
            int lab0 = -1;
            std::vector<Arc> probe;
            for (auto &g : order) {
                if (!own) break;
                if (g.part > 0) { own = false; break; }
                if (g.s0 < 0) continue;
                forward_row(g.s0, &probe);
                extract_own_fwd(g.s0, g.s0, g.s1, &probe, false);
                if (!probe.empty()) own = false;
                if (lab0 < 0) lab0 = g.lab0; else if (g.lab0 != lab0) own = false;
            }
        }
        plan->own_fwd.assign(2 * S + 4, 0.f);
        plan->own_bwd.assign(2 * S + 4, 0.f);
        plan->own_rows = own;
        if (own) merge = plan->num_pairs > 0;
        plan->fwd_merged = merge;
        int next_state = 0;
        for (auto &g : order) {
            Group fg, bg;
            if (g.part > 0 || (g.s0 < 0 && is_hub[(size_t)g.s1])) {
                // a PART of a hub's forward row: arcs [part*kPartArcs, ...) of the merged row + the target slot
                forward_row(g.s1, &hub_row);
                Segment f;
                const size_t a0 = std::min(hub_row.size(), (size_t)g.part * part_arcs), a1 = std::min(hub_row.size(), a0 + (size_t)part_arcs);
                for (size_t i = a0; i < a1; ++i) f.arcs.push_back(hub_row[i]);
                while (f.arcs.size() % kQuad != kQuad - 1) f.arcs.push_back(Arc{f.arcs.empty() ? (uint32_t)fid[(size_t)g.s1] : f.arcs.back().peer, 0.f});
                f.arcs.push_back(Arc{(uint32_t)fid[(size_t)g.s1], 0.f});   // last slot: the target row
                f.event = kEvPartial;
                f.rows = g.part == 0 ? 1 : 0;
                fg.first_state = bg.first_state = g.part == 0 ? fid[(size_t)g.s1] : next_state;
                fg.rows = bg.rows = f.rows;
                fg.pairs = bg.pairs = 0;
                fg.segs.push_back(std::move(f));
                if (g.part == 0) {
                    Segment b;
                    out_list(g.s1, &l1);
                    for (auto &e : l1) { b.arcs.push_back(Arc{(uint32_t)e.q, e.w}); b.w1.push_back(0.f); }
                    b.event = kEvRow;
                    b.rows = 1;
                    bg.segs.push_back(std::move(b));
                    next_state = fid[(size_t)g.s1] + 1;
                }
                fgroups.push_back(std::move(fg));
                bgroups.push_back(std::move(bg));
                continue;
            }
            fg.first_state = bg.first_state = g.s0 >= 0 ? fid[(size_t)g.s0] : fid[(size_t)g.s1];
            fg.rows = bg.rows = g.s0 >= 0 ? 2 : 1;
            fg.pairs = bg.pairs = g.s0 >= 0 ? 1 : 0;
            next_state = fg.first_state + fg.rows;
            if (g.s0 < 0) {
                Segment f, b;
                forward_row(g.s1, &f.arcs);
                if (own) extract_own_fwd(g.s1, -1, g.s1, &f.arcs, true);
                f.event = kEvRow;
                out_list(g.s1, &l1);
                if (own) extract_own_bwd(g.s1, -1, g.s1, &l1);
                for (auto &e : l1) { b.arcs.push_back(Arc{(uint32_t)e.q, e.w}); b.w1.push_back(0.f); }
                b.event = kEvRow;
                b.rows = 1;
                fg.segs.push_back(std::move(f));
                bg.segs.push_back(std::move(b));
            } else {
                Segment f0, f1, b;
                forward_row(g.s0, &f0.arcs); f0.event = kEvRowPos0;
                forward_row(g.s1, &f1.arcs); f1.event = kEvRowPos1;
                // backward: ONE segment for the pair; slot weights (w for p0, w1 for p1): shared arcs carry both
                out_list(g.s0, &l0);
                out_list(g.s1, &l1);
                if (own) {
                    extract_own_fwd(g.s0, g.s0, g.s1, &f0.arcs, true);   // (leaves f0 empty: checked above)
                    extract_own_fwd(g.s1, g.s0, g.s1, &f1.arcs, true);
                    extract_own_bwd(g.s0, g.s0, g.s1, &l0);
                    extract_own_bwd(g.s1, g.s0, g.s1, &l1);
                }
                size_t i = 0, j = 0;
                while (i < l0.size() || j < l1.size()) {
                    if (i < l0.size() && j < l1.size() && l0[i].q == l1[j].q && l0[i].wb == l1[j].wb) {
                        b.arcs.push_back(Arc{(uint32_t)l0[i].q, l0[i].w}); b.w1.push_back(l1[j].w); ++i; ++j;
                    } else if (j >= l1.size() || (i < l0.size() && (l0[i].q < l1[j].q || (l0[i].q == l1[j].q && l0[i].wb < l1[j].wb)))) {
                        b.arcs.push_back(Arc{(uint32_t)l0[i].q, l0[i].w}); b.w1.push_back(0.f); ++i;
                    } else {
                        b.arcs.push_back(Arc{(uint32_t)l1[j].q, 0.f}); b.w1.push_back(l1[j].w); ++j;
                    }
                }
                b.event = kEvRowPos1;
                b.rows = 2;
                if (merge) {   // one segment for the pair: p1's in-arcs, then (without own-row terms) p0's single arc in the last slot
                    if (!own) { f1.arcs.push_back(f0.arcs[0]); f1.tail = true; }
                    f1.event = kEvPairMerged;
                    f1.rows = 2;
                    f1.merged = true;
                    fg.segs.push_back(std::move(f1));
                } else {
                    fg.segs.push_back(std::move(f0)); fg.segs.push_back(std::move(f1));
                }
                bg.segs.push_back(std::move(b));
            }
            fgroups.push_back(std::move(fg));
            bgroups.push_back(std::move(bg));
        }
    };

    // largest total weight leaving a state (final weight included): the per-frame growth bound of a column sum
    {
        std::vector<double> out_sum((size_t)S0, 0.0);
        for (size_t a = 0; a < A0; ++a) out_sum[(size_t)fst.src[a]] += std::exp((double)fst.logw[a]);
        double G = 1.0;
        for (int q = 0; q < S0; ++q) {
            const float fw = fst.final_logw[(size_t)q];
            G = std::max(G, out_sum[(size_t)q] + (std::isinf(fw) ? 0.0 : std::exp((double)fw)));
        }
        const int e = (int)std::floor(61.0 - std::log2(G));
        if (e < 16) { *err = "den graph: a state's out-weights sum to " + std::to_string(G) + " -- not a probability-like graph"; return false; }
        plan->scale_exp = std::min(56, e);
    }
    plan->file_states = S0;
    plan->file_arcs = (int)A0;
    plan->num_states = (int)S;
    plan->num_labels = max_label + 1;
    plan->n_ctas = n_ctas;
    plan->n_warps = n_warps;

    // Phase 1: label-sorted order, to learn every group's cost in both passes.
    build(gk);
    const int G = (int)gk.size();
    auto seg_quads = [](const Segment &sg) { return std::max<int64_t>(1, ((int64_t)sg.arcs.size() + kQuad - 1) / kQuad); };
    // per-row costs in arc units, fitted to per-warp timelines (tools/timeline.py)
    constexpr int64_t kRowCostFwd = 5, kRowCostBwd = 8;
    std::vector<int64_t> cost((size_t)G, 0), cost_f((size_t)G, 0), cost_b((size_t)G, 0);
    for (int g = 0; g < G; ++g) {
        int64_t cf = 0, cb = 0;
        for (auto &sg : fgroups[(size_t)g].segs) cf += seg_quads(sg) * kQuad;
        for (auto &sg : bgroups[(size_t)g].segs) cb += seg_quads(sg) * kQuad;
        cost_f[(size_t)g] = cf + kRowCostFwd * fgroups[(size_t)g].rows;
        cost_b[(size_t)g] = cb + kRowCostBwd * fgroups[(size_t)g].rows;
        cost[(size_t)g] = cost_f[(size_t)g] + cost_b[(size_t)g];
    }
    // Phase 2: CTA tiles = contiguous ranges of the label-sorted order with equal total cost (both passes share the
    // tiles); inside a tile the groups are dealt to the warps longest-first (LPT), then each warp's groups are put
    // back in label order.  States are renumbered in that (tile, warp, label) order, which keeps every warp's rows
    // contiguous while balancing the warps to within one small group.
    // (floating parts of hub rows carry forward-pass work only: they are dealt over ALL tiles afterwards, to the tile
    // with the least forward load, instead of piling up in the tiles around their hub)
    std::vector<int64_t> prefix((size_t)G + 1, 0);
    for (int g = 0; g < G; ++g) prefix[(size_t)g + 1] = prefix[(size_t)g] + (gk[(size_t)g].part > 0 ? 0 : cost[(size_t)g]);
    std::vector<int> tile((size_t)n_ctas + 1, 0);
    for (int c = 1; c < n_ctas; ++c) {
        const int64_t target = (prefix[(size_t)G] * c + n_ctas / 2) / n_ctas;
        int g = (int)(std::lower_bound(prefix.begin(), prefix.end(), target) - prefix.begin());
        tile[(size_t)c] = std::min(std::max(g, tile[(size_t)c - 1]), G);
    }
    tile[(size_t)n_ctas] = G;
    std::vector<std::vector<int>> tile_groups((size_t)n_ctas);
    std::vector<int64_t> tile_fwd((size_t)n_ctas, 0);
    std::vector<int> floating;
    for (int c = 0; c < n_ctas; ++c)
        for (int g = tile[(size_t)c]; g < tile[(size_t)c + 1]; ++g) {
            if (gk[(size_t)g].part > 0) { floating.push_back(g); continue; }
            tile_groups[(size_t)c].push_back(g);
            for (auto &sg : fgroups[(size_t)g].segs) tile_fwd[(size_t)c] += seg_quads(sg) * kQuad;
        }
    for (int g : floating) {
        const int c = (int)(std::min_element(tile_fwd.begin(), tile_fwd.end()) - tile_fwd.begin());
        tile_groups[(size_t)c].push_back(g);
        for (auto &sg : fgroups[(size_t)g].segs) tile_fwd[(size_t)c] += seg_quads(sg) * kQuad;
    }
    std::vector<GroupKey> order;
    order.reserve((size_t)G);
    std::vector<int> chunk_group((size_t)n_ctas * n_warps + 1, 0);
    std::vector<std::vector<int>> bins((size_t)n_warps);
    std::vector<double> load_f((size_t)n_warps), load_b((size_t)n_warps);
    const bool balance_sum = getenv("CCB_BALANCE_SUM") != nullptr;
    std::vector<int> idx;
    for (int c = 0; c < n_ctas; ++c) {
        // Both passes walk the same warp -> rows assignment but their costs differ per group, and a frame of either
        // pass lasts as long as its slowest warp: balance the two loads as a vector (greedy: heaviest group first,
        // into the warp whose larger normalised load stays smallest), not their sum.
        idx = tile_groups[(size_t)c];
        double tot_f = 1e-9, tot_b = 1e-9;
        for (int g : idx) { tot_f += (double)cost_f[(size_t)g]; tot_b += (double)cost_b[(size_t)g]; }
        // CCB_BALANCE_SUM (tuning hook): balance the sum of the two passes' costs instead (the round-1 behaviour)
        auto nf = [&](int g) { return balance_sum ? (double)cost[(size_t)g] / (tot_f + tot_b) : (double)cost_f[(size_t)g] / tot_f; };
        auto nb = [&](int g) { return balance_sum ? (double)cost[(size_t)g] / (tot_f + tot_b) : (double)cost_b[(size_t)g] / tot_b; };
        std::stable_sort(idx.begin(), idx.end(), [&](int a, int b) { return std::max(nf(a), nb(a)) > std::max(nf(b), nb(b)); });
        for (auto &b : bins) b.clear();
        std::fill(load_f.begin(), load_f.end(), 0.0);
        std::fill(load_b.begin(), load_b.end(), 0.0);
        for (int g : idx) {
            int best = 0;
            double best_max = 1e300, best_sum = 1e300;
            for (int w = 0; w < n_warps; ++w) {
                const double f = load_f[(size_t)w] + nf(g), b = load_b[(size_t)w] + nb(g);
                const double m = std::max(f, b);
                if (m < best_max - 1e-12 || (m < best_max + 1e-12 && f + b < best_sum)) { best = w; best_max = m; best_sum = f + b; }
            }
            bins[(size_t)best].push_back(g);
            load_f[(size_t)best] += nf(g);
            load_b[(size_t)best] += nb(g);
        }
        // Local search on top of the greedy.  A warp's chunk is padded to whole batches of kChunkArcPad slots and the
        // grid barrier makes every frame of a pass wait for the longest chunk of the whole grid, so what counts is the
        // PADDED maximum per pass: move / swap groups out of the critical warps while that (then the number of warps
        // sitting at it, then the spread) improves.
        if (!balance_sum && idx.size() <= 320) {   // (big tiles: a group is a small fraction of a chunk, and the search is O(groups^2))
            std::vector<int64_t> sf((size_t)n_warps, 0), sb((size_t)n_warps, 0);   // slots per warp and pass
            auto slots_f = [&](int g) { int64_t c = 0; for (auto &sg : fgroups[(size_t)g].segs) c += seg_quads(sg) * kQuad; return c; };
            auto slots_b = [&](int g) { int64_t c = 0; for (auto &sg : bgroups[(size_t)g].segs) c += seg_quads(sg) * kQuad; return c; };
            for (int w = 0; w < n_warps; ++w)
                for (int g : bins[(size_t)w]) { sf[(size_t)w] += slots_f(g); sb[(size_t)w] += slots_b(g); }
            auto pad = [](int64_t x) { return (x + kChunkArcPad - 1) / kChunkArcPad; };
            struct Score { int64_t mx; int64_t at_max; int64_t sq; };
            auto score = [&]() {
                int64_t mf = 0, mb = 0;
                for (int w = 0; w < n_warps; ++w) { mf = std::max(mf, pad(sf[(size_t)w])); mb = std::max(mb, pad(sb[(size_t)w])); }
                Score sc{mf + mb, 0, 0};
                for (int w = 0; w < n_warps; ++w) {
                    sc.at_max += (pad(sf[(size_t)w]) == mf) + (pad(sb[(size_t)w]) == mb);
                    sc.sq += sf[(size_t)w] * sf[(size_t)w] + sb[(size_t)w] * sb[(size_t)w];
                }
                return sc;
            };
            auto better = [](const Score &a, const Score &b) {
                if (a.mx != b.mx) return a.mx < b.mx;
                if (a.at_max != b.at_max) return a.at_max < b.at_max;
                return a.sq < b.sq;
            };
            for (int iter = 0; iter < 300; ++iter) {
                const Score cur = score();
                int64_t mf = 0, mb = 0;
                for (int w = 0; w < n_warps; ++w) { mf = std::max(mf, pad(sf[(size_t)w])); mb = std::max(mb, pad(sb[(size_t)w])); }
                Score best = cur;
                int b_hw = -1, b_i = -1, b_w = -1, b_j = -1;
                for (int hw = 0; hw < n_warps; ++hw) {
                    if (pad(sf[(size_t)hw]) != mf && pad(sb[(size_t)hw]) != mb) continue;   // only critical warps give
                    for (int i = 0; i < (int)bins[(size_t)hw].size(); ++i) {
                        const int g = bins[(size_t)hw][(size_t)i];
                        const int64_t gf = slots_f(g), gb = slots_b(g);
                        for (int w = 0; w < n_warps; ++w) {
                            if (w == hw) continue;
                            for (int j = -1; j < (int)bins[(size_t)w].size(); ++j) {
                                const int64_t of = j < 0 ? 0 : slots_f(bins[(size_t)w][(size_t)j]), ob = j < 0 ? 0 : slots_b(bins[(size_t)w][(size_t)j]);
                                sf[(size_t)hw] += of - gf; sb[(size_t)hw] += ob - gb; sf[(size_t)w] += gf - of; sb[(size_t)w] += gb - ob;
                                const Score sc = score();
                                sf[(size_t)hw] -= of - gf; sb[(size_t)hw] -= ob - gb; sf[(size_t)w] -= gf - of; sb[(size_t)w] -= gb - ob;
                                if (better(sc, best)) { best = sc; b_hw = hw; b_i = i; b_w = w; b_j = j; }
                            }
                        }
                    }
                }
                if (b_hw < 0) break;
                const int g = bins[(size_t)b_hw][(size_t)b_i];
                const int o = b_j < 0 ? -1 : bins[(size_t)b_w][(size_t)b_j];
                const int64_t gf = slots_f(g), gb = slots_b(g), of = o < 0 ? 0 : slots_f(o), ob = o < 0 ? 0 : slots_b(o);
                sf[(size_t)b_hw] += of - gf; sb[(size_t)b_hw] += ob - gb; sf[(size_t)b_w] += gf - of; sb[(size_t)b_w] += gb - ob;
                if (o >= 0) { bins[(size_t)b_hw][(size_t)b_i] = o; bins[(size_t)b_w][(size_t)b_j] = g; }
                else { bins[(size_t)b_hw].erase(bins[(size_t)b_hw].begin() + b_i); bins[(size_t)b_w].push_back(g); }
            }
        }
        for (int w = 0; w < n_warps; ++w) {
            std::sort(bins[(size_t)w].begin(), bins[(size_t)w].end());   // label order (phase-1 index)
            chunk_group[(size_t)c * n_warps + w] = (int)order.size();
            for (int g : bins[(size_t)w]) order.push_back(gk[(size_t)g]);
        }
    }
    chunk_group[(size_t)n_ctas * n_warps] = (int)order.size();
    build(order);
    Layout(fgroups, (int)S, plan->state_label, plan->state_pos, n_ctas, n_warps, chunk_group, false, &plan->fwd);
    Layout(bgroups, (int)S, plan->state_label, plan->state_pos, n_ctas, n_warps, chunk_group, true, &plan->bwd);
    // the sampler's in-arc CSR, rows in the final numbering, each row's arcs in file order
    std::vector<int> sid_of_fid(S);
    for (size_t s = 0; s < S; ++s) sid_of_fid[(size_t)fid[s]] = (int)s;
    plan->in_off.assign(S + 1, 0);
    plan->in_src.clear(); plan->in_w.clear();
    plan->in_src.reserve(A); plan->in_w.reserve(A);
    for (size_t f = 0; f < S; ++f) {
        for (auto &a : in_s[(size_t)sid_of_fid[f]]) { plan->in_src.push_back(fid[(size_t)a.peer]); plan->in_w.push_back(a.w); }
        plan->in_off[f + 1] = (int)plan->in_src.size();
    }
    // the beam search's out-arc CSR: the same arcs by source, sorted by destination label, then destination
    plan->out_off.assign(S + 1, 0);
    for (int q : plan->in_src) ++plan->out_off[(size_t)q + 1];
    for (size_t s = 0; s < S; ++s) plan->out_off[s + 1] += plan->out_off[s];
    plan->out_dst.assign(plan->in_src.size(), 0);
    plan->out_w.assign(plan->in_src.size(), 0.f);
    {
        std::vector<int> fill(plan->out_off.begin(), plan->out_off.end() - 1);
        for (size_t f = 0; f < S; ++f)
            for (int i = plan->in_off[f]; i < plan->in_off[f + 1]; ++i) {
                const int k = fill[(size_t)plan->in_src[(size_t)i]]++;
                plan->out_dst[(size_t)k] = (int)f;
                plan->out_w[(size_t)k] = plan->in_w[(size_t)i];
            }
        std::vector<std::pair<int, int>> row;
        std::vector<float> roww;
        for (size_t s = 0; s < S; ++s) {
            const int b = plan->out_off[s], e = plan->out_off[s + 1];
            row.clear();
            for (int i = b; i < e; ++i) row.emplace_back(i, plan->out_dst[(size_t)i]);
            std::sort(row.begin(), row.end(), [&](const std::pair<int, int> &x, const std::pair<int, int> &y) {
                const int lx = plan->state_label[(size_t)x.second], ly = plan->state_label[(size_t)y.second];
                return lx != ly ? lx < ly : (x.second != y.second ? x.second < y.second : x.first < y.first);
            });
            roww.clear();
            for (auto &r : row) roww.push_back(plan->out_w[(size_t)r.first]);
            for (int i = b; i < e; ++i) {
                plan->out_dst[(size_t)i] = row[(size_t)(i - b)].second;
                plan->out_w[(size_t)i] = roww[(size_t)(i - b)];
            }
        }
    }
    return true;
}

namespace {
// the out-arc of p into a state of label c (-1: none); the labels of a state's out-arcs are sorted
int OutArcTo(const DenPlan &g, int p, int c) {
    if (p < 0) return -1;
    int lo = g.out_off[(size_t)p], hi = g.out_off[(size_t)p + 1];
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (g.state_label[(size_t)g.out_dst[(size_t)mid]] < c) lo = mid + 1; else hi = mid;
    }
    return lo < g.out_off[(size_t)p + 1] && g.state_label[(size_t)g.out_dst[(size_t)lo]] == c ? g.out_dst[(size_t)lo] : -1;
}

std::string StateName(const DenPlan &g, int q) {
    return std::to_string(q) + " (file state " + std::to_string(g.orig_state[(size_t)q]) + ", label " +
           std::to_string(g.state_label[(size_t)q]) + ")";
}
}  // namespace

bool CheckCtcShape(const DenPlan &g, std::string *err) {
    const int S = g.num_states;
    for (int p = 0; p < S; ++p)
        for (int i = g.out_off[(size_t)p] + 1; i < g.out_off[(size_t)p + 1]; ++i) {
            const int a = g.out_dst[(size_t)i - 1], b = g.out_dst[(size_t)i];
            if (g.state_label[(size_t)a] == g.state_label[(size_t)b]) {
                *err = "den graph is not CTC-shaped: state " + StateName(g, p) + " has out-arcs into two states of label " +
                       std::to_string(g.state_label[(size_t)a]) + ": " + StateName(g, a) + " and " + StateName(g, b);
                return false;
            }
        }
    // a slot in state q that reads label c again (the blank slot: blank; the token slot: its token) must stay in q
    auto stays = [&](int q, int c, const char *slot) {
        const int d = OutArcTo(g, q, c);
        if (d < 0 || d == q) return true;
        *err = std::string("den graph is not CTC-shaped: the ") + slot + " slot in state " + StateName(g, q) +
               " moves to state " + StateName(g, d) + " on label " + std::to_string(c) + " instead of staying";
        return false;
    };
    // signature of a prefix: (blank-slot state, token-slot state), -1 = empty; the last token is the token-slot state's label
    auto key = [](int b, int t) { return ((uint64_t)(uint32_t)(b + 1) << 32) | (uint32_t)(t + 1); };
    std::unordered_set<uint64_t> seen;
    std::vector<std::pair<int, int>> queue;
    if (!stays(g.start, 0, "blank")) return false;
    queue.emplace_back(g.start, -1);
    seen.insert(key(g.start, -1));
    std::vector<int> labels;
    for (size_t head = 0; head < queue.size(); ++head) {
        const int b = queue[head].first, t = queue[head].second;
        const int last = t >= 0 ? g.state_label[(size_t)t] : -1;
        labels.clear();
        for (int q : {b, t})
            if (q >= 0)
                for (int i = g.out_off[(size_t)q]; i < g.out_off[(size_t)q + 1]; ++i) labels.push_back(g.state_label[(size_t)g.out_dst[(size_t)i]]);
        std::sort(labels.begin(), labels.end());
        labels.erase(std::unique(labels.begin(), labels.end()), labels.end());
        for (int c : labels) {
            if (c == 0) continue;
            const int d1 = OutArcTo(g, b, c), d2 = c != last ? OutArcTo(g, t, c) : -1;
            if (d1 >= 0 && d2 >= 0 && d1 != d2) {
                *err = "den graph is not CTC-shaped: the blank slot in state " + StateName(g, b) + " and the token slot in state " +
                       StateName(g, t) + " of one prefix step into different states " + StateName(g, d1) + " and " +
                       StateName(g, d2) + " on token " + std::to_string(c);
                return false;
            }
            const int nt = d1 >= 0 ? d1 : d2;
            if (nt < 0) continue;
            if (!stays(nt, c, "token")) return false;
            const int nb = OutArcTo(g, nt, 0);
            if (nb >= 0 && !stays(nb, 0, "blank")) return false;
            if (seen.insert(key(nb, nt)).second) queue.emplace_back(nb, nt);
        }
    }
    return true;
}

// ---- launch of the persistent den kernels (den_launch.h) ----
bool ChooseDenLaunch(const DenGraphShape &g, int Npad, bool backward, int smem_optin, const DenHooks &hooks, DenLaunch *out,
                     std::string *why) {
    if (g.n_warps * 32 != kDenThreads || Npad > kDenThreads || (Npad != kSmallLanes && Npad != 32 && Npad != 64 && (Npad <= 0 || Npad % 128))) {
        *why = "den: no kernel for " + std::to_string(Npad) + " lanes at " + std::to_string(g.n_warps) + " warps per CTA (16, N <= 512)";
        return false;
    }
    const DenPassShape &pass = backward ? g.bwd : g.fwd;
    auto up128 = [](size_t x) { return (x + 127) & ~(size_t)127; };
    const size_t budget = (size_t)smem_optin > 2048 ? (size_t)smem_optin - 1024 : 0, nw = (size_t)g.n_warps;
    DenLaunch L;
    L.tile_rows = pass.max_tile_rows;   // and backward, the label accumulator in shared memory if the CTA's label range is small
    L.gacc_rows = backward && (size_t)pass.max_tile_labels * Npad * 4 <= 64 * 1024 ? pass.max_tile_labels : 0;
    L.arcs_off = backward ? BwdArcsOff(Npad, L.gacc_rows, L.tile_rows) : FwdArcsOff(Npad, L.tile_rows);
    // Tiers by graph size, for batches of more than 16 utterances.  (1) The whole arc stream in shared memory (8 bytes per
    // forward slot, 12 per backward slot), rows gathered into registers: on an H100 this beats staging the rows by one TMA
    // copy each at every batch width (N = 32 / 64 / 128, T = 1500, 1.02 M arcs: 46.7 / 79.9 / 160.1 ms per step against
    // 56.0 / 87.5 / 175.1 ms, 700 W, 1980 MHz); (2) backward only: offsets + first weights in shared memory, second weights
    // streamed from L2, or the streamed-arc TMA tier below; (3) everything from L2.
    // Small batches: the arc stream must fit NEXT TO the small-batch rings; the 12-byte backward form gives way to the 8-byte
    // one when only that leaves them room.
    const bool small = Npad == kSmallLanes;
    const size_t small_extra = small ? 128 + nw * (kSmallRingWarpBytes + kSmallBarWarpBytes + kSmallW1WarpBytes) : 0;
    bool w1_smem = backward && !hooks.w1_in_global;
    size_t arc_bytes = (size_t)pass.max_tile_arcs * (w1_smem ? 12 : sizeof(Arc));
    if (w1_smem && L.arcs_off + arc_bytes + small_extra > budget) { w1_smem = false; arc_bytes = (size_t)pass.max_tile_arcs * sizeof(Arc); }
    const bool smem_arcs = L.arcs_off + arc_bytes + small_extra <= budget && !hooks.arcs_in_global;
    if (small) {   // one utterance per lane, 16 lanes per row; needs the arc tile resident and no hub rows
        L.tier = kTierSmall; L.lanes_per_row = kSmallLanes; L.batch = kSmallRows; L.w1_smem = w1_smem;
        L.ring_off = up128(L.arcs_off + (smem_arcs ? arc_bytes : 0)); L.bar_off = L.ring_off + nw * kSmallRingWarpBytes;
        L.w1_off = SmallW1Off((uint32_t)L.bar_off, g.n_warps); L.total = L.w1_off + nw * kSmallW1WarpBytes;   // (forward too)
        *out = L;
        if (smem_arcs && L.total <= budget && g.n_hubs == 0 && !hooks.no_tma) return true;
        *why = "den: no small-batch kernels for this graph/device (smem " + std::to_string(L.total) + "/" + std::to_string(budget) + ")";
        return false;
    }
    // utterances per lane: the widest row segment the batch allows, except that the backward pass (two accumulators per
    // utterance) spills at 4 -- it walks 64-utterance groups instead
    L.U = Npad >= 128 ? (backward ? 2 : 4) : Npad / 32;
    // Streamed-arc TMA tier, BACKWARD pass only: the stream does not fit (or the test hook says so) but the graph carries the
    // transposed copy.  The forward pass of such graphs keeps the register gathers with the arcs read from L2: its 8-byte
    // slots would make 128-byte bulk copies, one per 16 rows.
    if (backward && !(smem_arcs && w1_smem) && g.streamed_quads && g.n_hubs == 0 && !hooks.no_tma) {
        DenLaunch S = L;
        S.tier = kTierStreamed; S.batch = kStreamRows;
        S.ring_off = up128(S.arcs_off); S.bar_off = S.ring_off + nw * StreamRingWarpBytes(S.U);
        S.abar_off = S.bar_off + nw * kStreamBarWarpBytes; S.aring_off = up128(S.abar_off + nw * kArcBarWarpBytes);
        S.total = S.aring_off + nw * kArcRingWarpBytes;
        if (S.total <= budget) { *out = S; return true; }
    }
    L.tier = smem_arcs ? kTierShared : kTierGlobal; L.w1_smem = smem_arcs && w1_smem;
    L.batch = backward ? kBwdBatch : FwdBatch(L.U); L.total = L.arcs_off + (smem_arcs ? arc_bytes : 0);
    // Own rows on chip: each warp reads back the rows it wrote one frame earlier (the own-row terms, 2 per pair) from a
    // [tile_rows][Npad] copy behind the arc tile instead of from L2, where it fits (N = 64 at 132 CTAs: 78 KB)
    const size_t own_off = (L.total + 15) & ~(size_t)15, own_bytes = (size_t)L.tile_rows * Npad * 4;
    if (g.own_rows && !hooks.own_in_l2 && own_off + own_bytes <= budget) {
        L.own_smem = true; L.own_off = own_off; L.total = own_off + own_bytes;
    }
    *out = L;
    return true;
}

bool SmallBatchOk(const DenGraphShape &g, int smem_optin, const DenHooks &hooks) {
    DenLaunch L;
    std::string why;
    return ChooseDenLaunch(g, kSmallLanes, false, smem_optin, hooks, &L, &why) && ChooseDenLaunch(g, kSmallLanes, true, smem_optin, hooks, &L, &why);
}

DenGraphShape ShapeOf(const DenPlan &plan, const DenHooks &hooks) {
    const int n_hubs = (int)plan.hub_states.size();
    return {{plan.fwd.max_tile_arcs, plan.fwd.max_tile_rows, plan.fwd.max_tile_labels},
            {plan.bwd.max_tile_arcs, plan.bwd.max_tile_rows, plan.bwd.max_tile_labels}, n_hubs, plan.n_warps,
            n_hubs == 0 && !hooks.no_tma && (hooks.arcs_in_global || LargeGraphTiers(plan.bwd.max_tile_arcs)), plan.own_rows};
}

}  // namespace ccb
