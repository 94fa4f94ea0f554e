// CTC prefix beam search over the logits (plain CTC) or over the den graph (the CTC-CRF posterior), N-best per utterance.
//
// One CTA per utterance, one launch for the batch.  The beam holds up to B prefixes; each is a trie node with two slots,
// "ends in blank" and "ends in its last token", each a log mass in fp64 and, in crf mode, the den state every path of the
// slot is in (CheckCtcShape, den_graph.cc, guarantees that there is one).  Each frame (DESIGN.md §7 "Prefix beam search"):
//   1. the y row is staged in shared memory and its cutoff_top_n largest entries (ties: lower id) are the frame's tokens;
//   2. every entry r yields the candidates "stay" (r itself: blank from both slots, the repeat of its last token from the
//      token slot) and "r + c" for every frame token c and its own last token (from the blank slot, and from the token slot
//      when c differs from the last token); den arcs are found by binary search in the label-sorted out-arcs of a state;
//   3. an extension whose prefix is itself in the beam is merged into that entry's stay candidate (a shared-memory map of
//      (parent rank, token) -> child, then a fixed-order sum: no atomics);
//   4. the candidates are ranked by (mass desc, key asc), key = (rank of the parent entry, token), -1 for a stay; they are
//      generated in chunks and each chunk is bitonic-sorted together with the best B so far;
//   5. the B best become the next beam; an extension's trie node is looked up in the open-addressing hash on (parent, token)
//      and created if missing, new node ids in rank order.
// After the last frame every entry gets its final score (crf: plus log final of each slot's state), the entries are ranked
// by it, and the trie is walked back to write tokens, the frame at which each token's node was created, lengths and scores.
// With a token n-gram LM (plain mode, the LM template flag; DESIGN.md §7 "N-gram LM fusion") each entry also carries an LM
// state and LM part, an extension's rank adds alpha ln P(c | state) + beta (a back-off walk over the LM's tables), and the
// final score adds alpha ln P(</s> | state).
#include <cmath>

#include "beam_common.cuh"
#include "common.cuh"

namespace ccb {

namespace {

constexpr int kThreads = 512;
constexpr int kChunkSort = 2048;    // candidates + running best per bitonic sort (at least; a larger vocabulary widens it)
constexpr int kMapSlots = 256;      // (parent rank, token) -> child map, at most kBeamMax keys

// per utterance: parent, token, first frame and beam rank of every node, then the hash table (node ids, -1 = empty)
__host__ __device__ __forceinline__ size_t UttBytes(int T, int B) {
    return Up256((4 * NodeCap(T, B) + HashSlots(T, B)) * sizeof(int));
}

struct Graph {   // crf mode: the split den graph's out-arc CSR (DenPlan::out_*), labels and finals
    const int *out_off, *out_dst, *state_label;
    const float *out_w, *final_lin;
    int start;
};

// log w of the out-arc of state s into a state of label c, *dst its destination; -inf and -1 if there is none.  Plain mode
// (crf false): every step is allowed with weight 1 and there are no states.
__device__ __forceinline__ double Step(bool crf, const Graph &g, int s, int c, int *dst) {
    *dst = -1;
    if (!crf) return 0.0;
    if (s < 0) return kNegInf;
    int lo = g.out_off[s];
    const int end = g.out_off[s + 1];
    int hi = end;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (g.state_label[g.out_dst[mid]] < c) lo = mid + 1; else hi = mid;
    }
    if (lo < end && g.state_label[g.out_dst[lo]] == c) {
        *dst = g.out_dst[lo];
        return log((double)g.out_w[lo]);
    }
    return kNegInf;
}

struct Beam {    // one beam in shared memory
    int *node, *last, *sb, *st, *par;   // par: rank of the parent entry when this entry's last token extends it this frame
    double *mb, *mt;
};

struct Slots {
    double mb, mt;
    int sb, st;
};

// The mass entry r sends into prefix r + c (token slot): from its blank slot, and from its token slot unless c repeats
// its last token.
__device__ __forceinline__ double ExtIn(bool crf, const Graph &g, const Beam &o, int r, int c, int *dst) {
    int d1, d2;
    const double a = o.mb[r] + Step(crf, g, o.sb[r], c, &d1);
    const double b = c != o.last[r] ? o.mt[r] + Step(crf, g, o.st[r], c, &d2) : (d2 = -1, kNegInf);
    *dst = a > kNegInf ? d1 : d2;
    return lse(a, b);
}

// Candidate "stay" of entry r: blank from both slots, the repeat of the last token, and (when par >= 0) the extension of
// the parent entry that this prefix is.
__device__ __forceinline__ Slots Stay(bool crf, const Graph &g, const Beam &o, int r, const float *yrow) {
    Slots s;
    int d1, d2;
    const double a = o.mb[r] + Step(crf, g, o.sb[r], 0, &d1);
    const double b = o.mt[r] + Step(crf, g, o.st[r], 0, &d2);
    const double bin = lse(a, b);
    s.sb = bin > kNegInf ? (a > kNegInf ? d1 : d2) : -1;
    s.mb = bin > kNegInf ? bin + (double)yrow[0] : kNegInf;
    const int l = o.last[r];
    s.mt = kNegInf;
    s.st = -1;
    if (l >= 1) {
        int d3, d4 = -1;
        const double rep = o.mt[r] + Step(crf, g, o.st[r], l, &d3);
        const double ext = o.par[r] >= 0 ? ExtIn(crf, g, o, o.par[r], l, &d4) : kNegInf;
        const double tin = lse(rep, ext);
        if (tin > kNegInf) {
            s.mt = tin + (double)yrow[l];
            s.st = rep > kNegInf ? d3 : d4;
        }
    }
    return s;
}

__device__ __forceinline__ unsigned MapHash(int key) { return ((unsigned)key * 0x9E3779B1u) >> 24; }   // kMapSlots = 256

struct Params {
    Graph g;
    bool crf;
    const void *y;
    int y_dtype;
    int N, T, V, B, topn, psort;
    const int *len;
    char *ws;
    int *tokens, *lengths, *timesteps;
    float *scores;
    // the LM instantiation only (kept last: the fields above keep their offsets in both instantiations)
    NGramDev lm;
    double alpha, beta;
};

// What an extension by token c from LM state s adds to a prefix's LM part: alpha ln P(c | s) + beta; *dst the state after
// c.  alpha = 0 does not consult the LM.
__device__ __forceinline__ double LmTerm(const Params &P, int s, int c, int *dst) {
    if (P.alpha == 0.0) { *dst = s; return P.beta; }
    // (rounded operation by operation, not fused, so that a restatement in numpy reproduces it)
    return __dadd_rn(__dmul_rn(P.alpha, __dmul_rn(LmLog10(P.lm, s, P.lm.tok2word[c], dst), kLn10)), P.beta);
}

// LM: the token n-gram LM fused in (plain mode only).  Each entry then also carries its LM state and LM part (the sum of
// its extensions' LmTerm); a candidate ranks by its acoustic mass plus its prefix's LM part, and after the last frame each
// entry adds alpha ln P(</s> | state).  The instantiation without it is the search without an LM.
template <bool LM>
__global__ void __launch_bounds__(kThreads) beam_search_kernel(const Params P) {
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ int s_nb, s_next, s_count;
    const int n = blockIdx.x, tid = threadIdx.x;
    const int V = P.V, B = P.B, T = P.T;
    const bool crf = P.crf;
    const Graph &g = P.g;
    // shared memory: sort buffer, y row, token flags and list, two beams, the child map, winner scratch
    double *sort_m = reinterpret_cast<double *>(smem);
    int *sort_k = reinterpret_cast<int *>(sort_m + P.psort);
    float *yrow = reinterpret_cast<float *>(sort_k + P.psort);
    int *flag = reinterpret_cast<int *>(yrow + V);
    int *toks = flag + V;
    double *bd = reinterpret_cast<double *>(toks + V + (V & 1));
    Beam bm[2];
    for (int i = 0; i < 2; ++i) { bm[i].mb = bd + (2 * i) * B; bm[i].mt = bd + (2 * i + 1) * B; }
    int *bi = reinterpret_cast<int *>(bd + 4 * B);
    for (int i = 0; i < 2; ++i) {
        bm[i].node = bi + (5 * i) * B; bm[i].last = bi + (5 * i + 1) * B; bm[i].sb = bi + (5 * i + 2) * B;
        bm[i].st = bi + (5 * i + 3) * B; bm[i].par = bi + (5 * i + 4) * B;
    }
    int *map = bi + 10 * B;
    int *wnode = map + kMapSlots;
    // LM: the LM part (fp64) and LM state of the entries of both beams
    double *lmd = reinterpret_cast<double *>(wnode + B + (B & 1));
    int *lsd = reinterpret_cast<int *>(lmd + 2 * B);

    // the utterance's trie: node 0 is the root (the empty prefix)
    const size_t cap = NodeCap(T, B), hslots = HashSlots(T, B);
    int *t_parent = reinterpret_cast<int *>(P.ws + (size_t)n * UttBytes(T, B));
    int *t_tok = t_parent + cap, *t_frame = t_tok + cap, *t_rank = t_frame + cap, *hash = t_rank + cap;
    for (size_t i = tid; i < hslots; i += blockDim.x) hash[i] = -1;
    for (int c = tid; c < V; c += blockDim.x) { flag[c] = 1; toks[c] = c; }
    const int ln = P.len[n];
    const int topn = P.topn;
    if (tid == 0) {
        t_parent[0] = -1; t_tok[0] = -1; t_frame[0] = -1; t_rank[0] = 0;
        bm[0].node[0] = 0; bm[0].last[0] = -1; bm[0].par[0] = -1;
        bm[0].mb[0] = 0.0; bm[0].sb[0] = crf ? g.start : -1;
        bm[0].mt[0] = kNegInf; bm[0].st[0] = -1;
        s_nb = 1; s_next = 1;
        if constexpr (LM) { lmd[0] = 0.0; lsd[0] = P.lm.bos; }
    }
    __syncthreads();
    int cur = 0;
    const int per = topn + 2;   // candidates per entry: stay, the frame tokens, its own last token
    for (int t = 0; t < ln; ++t) {
        Beam &o = bm[cur], &w = bm[cur ^ 1];
        const double *lmo = lmd + cur * B;
        const int *lso = lsd + cur * B;
        const int nb = s_nb;
        // 1. the y row and the frame's tokens
        const long yb = ((long)n * T + t) * V;
        for (int c = tid; c < V; c += blockDim.x) yrow[c] = load_y(P.y, P.y_dtype, yb + c);
        for (int i = tid; i < kMapSlots; i += blockDim.x) map[i] = -1;
        __syncthreads();
        if (topn < V) {
            const int pv = Pow2Ceil(V);
            for (int i = tid; i < pv; i += blockDim.x) {
                sort_m[i] = i < V ? (double)yrow[i] : kNegInf;
                sort_k[i] = i < V ? i : 0x7fffffff;
                if (i < V) flag[i] = 0;
            }
            __syncthreads();
            BitonicSort(sort_m, sort_k, pv);
            for (int i = tid; i < topn; i += blockDim.x) { toks[i] = sort_k[i]; flag[sort_k[i]] = 1; }
            __syncthreads();
        }
        // the entries whose prefix extends another entry of the beam by a token that entry extends by this frame
        for (int r = tid; r < nb; r += blockDim.x) {
            const int node = o.node[r], parent = t_parent[node];
            const int pr = parent >= 0 ? t_rank[parent] : -1;
            const int c = o.last[r];
            o.par[r] = -1;
            if (pr >= 0 && (flag[c] || c == o.last[pr])) {
                o.par[r] = pr;
                const int key = pr * (V + 1) + c;
                unsigned h = MapHash(key);
                while (atomicCAS(&map[h], -1, key) != -1) h = (h + 1) & (kMapSlots - 1);
            }
        }
        __syncthreads();
        // 2-4. candidates in chunks, each sorted together with the best B so far (slots [0, B) of the sort buffer)
        for (int i = tid; i < B; i += blockDim.x) { sort_m[i] = kNegInf; sort_k[i] = 0x7fffffff; }
        const int total = nb * per;
        const int chunk = P.psort - B;
        for (int c0 = 0; c0 < total; c0 += chunk) {
            const int cnt = min(chunk, total - c0);
            const int ps = Pow2Ceil(B + cnt);
            for (int i = tid; i < ps - B; i += blockDim.x) {
                double m = kNegInf;
                int key = 0x7fffffff;
                if (i < cnt) {
                    const int idx = c0 + i, r = idx / per, j = idx % per;
                    if (j == 0) {
                        const Slots s = Stay(crf, g, o, r, yrow);
                        m = lse(s.mb, s.mt);
                        if constexpr (LM) m += lmo[r];
                        key = r * (V + 1);
                    } else {
                        const int c = j <= topn ? toks[j - 1] : o.last[r];
                        const bool valid = c >= 1 && (j <= topn || !flag[c]);
                        bool merged = false;
                        if (valid) {
                            const int mk = r * (V + 1) + c;
                            for (unsigned h = MapHash(mk); map[h] != -1; h = (h + 1) & (kMapSlots - 1))
                                if (map[h] == mk) { merged = true; break; }
                        }
                        if (valid && !merged) {
                            int d;
                            const double ein = ExtIn(crf, g, o, r, c, &d);
                            m = ein > kNegInf ? ein + (double)yrow[c] : kNegInf;
                            if constexpr (LM) {
                                int ls;
                                if (m > kNegInf) m += lmo[r] + LmTerm(P, lso[r], c, &ls);
                            }
                            key = r * (V + 1) + c + 1;
                        }
                    }
                    if (!(m > kNegInf)) { m = kNegInf; key = 0x7fffffff; }
                }
                sort_m[B + i] = m;
                sort_k[B + i] = key;
            }
            __syncthreads();
            BitonicSort(sort_m, sort_k, ps);
        }
        // 5. the next beam, in rank order; trie nodes of the extensions looked up, missing ones created in rank order
        if (tid == 0) {
            int k = 0;
            while (k < B && sort_m[k] > kNegInf) ++k;
            s_count = k;
        }
        __syncthreads();
        const int nb2 = s_count;
        for (int k = tid; k < nb2; k += blockDim.x) {
            const int key = sort_k[k], r = key / (V + 1), c = key % (V + 1) - 1;
            if (c < 0) {
                const Slots s = Stay(crf, g, o, r, yrow);
                w.node[k] = o.node[r]; w.last[k] = o.last[r];
                w.mb[k] = s.mb; w.sb[k] = s.sb; w.mt[k] = s.mt; w.st[k] = s.st;
                wnode[k] = -2;
                if constexpr (LM) { lmd[(cur ^ 1) * B + k] = lmo[r]; lsd[(cur ^ 1) * B + k] = lso[r]; }
            } else {
                int d;
                const double ein = ExtIn(crf, g, o, r, c, &d);
                const int parent = o.node[r];
                w.last[k] = c;
                w.mb[k] = kNegInf; w.sb[k] = -1; w.mt[k] = ein + (double)yrow[c]; w.st[k] = d;
                if constexpr (LM) {
                    int ls;
                    lmd[(cur ^ 1) * B + k] = lmo[r] + LmTerm(P, lso[r], c, &ls);
                    lsd[(cur ^ 1) * B + k] = ls;
                }
                int found = -1;
                for (unsigned h = TrieHash(parent, c, hslots);; h = (h + 1) & (unsigned)(hslots - 1)) {
                    const int x = hash[h];
                    if (x < 0) break;
                    if (t_parent[x] == parent && t_tok[x] == c) { found = x; break; }
                }
                w.node[k] = found;
                wnode[k] = found >= 0 ? -2 : parent;
            }
        }
        __syncthreads();
        if (tid == 0) {
            int next = s_next;
            for (int k = 0; k < nb2; ++k)
                if (wnode[k] != -2) { w.node[k] = next++; }
            s_next = next;
        }
        __syncthreads();
        for (int k = tid; k < nb2; k += blockDim.x) {
            if (wnode[k] == -2) continue;
            const int x = w.node[k], parent = wnode[k], c = w.last[k];
            t_parent[x] = parent; t_tok[x] = c; t_frame[x] = t; t_rank[x] = -1;
            unsigned h = TrieHash(parent, c, hslots);
            while (atomicCAS(&hash[h], -1, x) != -1) h = (h + 1) & (unsigned)(hslots - 1);
        }
        for (int r = tid; r < nb; r += blockDim.x) t_rank[o.node[r]] = -1;
        __syncthreads();
        for (int k = tid; k < nb2; k += blockDim.x) t_rank[w.node[k]] = k;
        if (tid == 0) s_nb = nb2;
        cur ^= 1;
        __syncthreads();
    }
    // final scores (crf: plus log final of each slot's state), ranked (score desc, beam rank asc), the trie walked back
    const Beam &o = bm[cur];
    const int nb = s_nb;
    double *fs = sort_m;
    for (int k = tid; k < B; k += blockDim.x) {
        double s = kNegInf;
        if (k < nb) {
            if (crf) {
                const double a = o.sb[k] >= 0 ? o.mb[k] + log((double)g.final_lin[o.sb[k]]) : kNegInf;
                const double b = o.st[k] >= 0 ? o.mt[k] + log((double)g.final_lin[o.st[k]]) : kNegInf;
                s = lse(a, b);
            } else {
                s = lse(o.mb[k], o.mt[k]);
            }
            if constexpr (LM) {
                if (s > kNegInf) {
                    int d;
                    const double *lmf = lmd + cur * B;
                    const int *lsf = lsd + cur * B;
                    s += lmf[k] + (P.alpha != 0.0 ? __dmul_rn(P.alpha, __dmul_rn(LmLog10(P.lm, lsf[k], P.lm.eos, &d), kLn10)) : 0.0);
                }
            }
        }
        fs[k] = s > kNegInf ? s : kNegInf;
    }
    __syncthreads();
    if (tid == 0) {
        int c = 0;
        for (int k = 0; k < nb; ++k) c += fs[k] > kNegInf;
        s_count = c;
    }
    __syncthreads();
    const int nfin = s_count;
    const size_t row0 = (size_t)n * B;
    for (int k = tid; k < B; k += blockDim.x) {
        int pos = k;                   // rows nfin.. are written by the threads of the entries without a finite score
        int node = -1;
        if (k < nb && fs[k] > kNegInf) {
            pos = 0;
            for (int j = 0; j < nb; ++j) pos += Before(fs[j], j, fs[k], k) && fs[j] > kNegInf;
            node = o.node[k];
        } else {
            int below = 0;             // the entries before k without a finite score take rows nfin, nfin+1, ...
            for (int j = 0; j < k; ++j) below += !(j < nb && fs[j] > kNegInf);
            pos = nfin + below;
        }
        int *tk = P.tokens + (row0 + pos) * T, *ts = P.timesteps + (row0 + pos) * T;
        int L = -1;
        if (node >= 0) {
            L = 0;
            for (int x = node; x > 0; x = t_parent[x]) ++L;
            int i = L;
            for (int x = node; x > 0; x = t_parent[x]) { --i; tk[i] = t_tok[x]; ts[i] = t_frame[x]; }
        }
        for (int i = max(L, 0); i < T; ++i) { tk[i] = -1; ts[i] = -1; }
        P.lengths[row0 + pos] = L;
        P.scores[row0 + pos] = node >= 0 ? (float)fs[k] : -INFINITY;
    }
}

}  // namespace

size_t BeamWsBytes(int N, int T, int B) { return (size_t)N * UttBytes(T, B); }

int LaunchBeamSearch(const DeviceGraph *dg, const void *y, int y_dtype, int N, int T, int V, const int *len, int B, int topn,
                     void *ws, int *tokens, int *lengths, int *timesteps, float *scores, cudaStream_t stream,
                     const NGramDev *lm, double alpha, double beta) {
    Params p;
    p.lm = lm ? *lm : NGramDev{};
    p.alpha = alpha; p.beta = beta;
    p.crf = dg != nullptr;
    p.g = Graph{};
    if (dg) {
        p.g.out_off = dg->out_off; p.g.out_dst = dg->out_dst; p.g.state_label = dg->state_label;
        p.g.out_w = dg->out_w; p.g.final_lin = dg->final_lin; p.g.start = dg->start;
    }
    p.y = y; p.y_dtype = y_dtype; p.N = N; p.T = T; p.V = V; p.B = B; p.topn = topn; p.len = len;
    p.psort = Pow2Ceil(V) > kChunkSort ? Pow2Ceil(V) : kChunkSort;
    p.ws = reinterpret_cast<char *>(ws);
    p.tokens = tokens; p.lengths = lengths; p.timesteps = timesteps; p.scores = scores;
    // (the LM instantiation: + the LM part and state of the entries of both beams, 24 B bytes)
    const size_t smem = (size_t)p.psort * (sizeof(double) + sizeof(int)) + (size_t)V * 3 * sizeof(int) + sizeof(int) * (V & 1) +
                        (size_t)B * 4 * sizeof(double) + ((size_t)B * 11 + kMapSlots) * sizeof(int) +
                        (lm ? sizeof(int) * (B & 1) + (size_t)B * 2 * (sizeof(double) + sizeof(int)) : 0);
    auto kernel = lm ? beam_search_kernel<true> : beam_search_kernel<false>;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    kernel<<<N, kThreads, smem, stream>>>(p);
    CountLaunch();
    return (int)cudaGetLastError();
}

}  // namespace ccb
