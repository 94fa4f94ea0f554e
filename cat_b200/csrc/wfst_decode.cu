// 1-best word decoding through a TLG decoding graph (wfst.h): a frame-synchronous Viterbi beam search, one CTA per
// utterance, the frame loop inside the kernel, one launch for the batch (DESIGN.md §7 "TLG decoding").
//
// Search costs are fp32, rounded operation by operation (__fadd_rn / __fmul_rn, no contraction), so that a numpy float32
// restatement reproduces every decision.  With acs = acwt / lmwt and wps = wip / lmwt:
//   emitting arc a from a token of cost c:  ((c + w_a) + (-acs * y[t][tok_a])) + (olabel_a != 0 ? wps : 0)
//   epsilon arc a:                          (c + w_a) + (olabel_a != 0 ? wps : 0)
// Each frame:
//   1. every kept token of the previous layer expands along its emitting arcs; best_e = the smallest candidate cost and
//      cutoff = best_e + beam (a first pass over the arcs);
//   2. the candidates within the cutoff are inserted (a second pass) into an open-addressing hash of state -> packed
//      (ordered cost bits, file arc id), updated with a 64-bit atomicMin: the winner is the smallest (cost, arc id)
//      whatever the thread order;
//   3. epsilon closure by increasing epsilon level (the longest epsilon path into a state), so that a state's token is
//      final before its epsilon arcs are relaxed; a relaxed cost enters only within the cutoff;
//   4. the kept tokens are the max_active smallest by (cost, state): an exact radix select on the 64-bit key
//      (ordered cost bits, state), 8 bits per pass.
// Each kept token then writes a record: the index of its predecessor token in the previous layer and the file ids of the
// arcs taken since (its epsilon chain back to the emitting arc, at most L + 1), so words on epsilon chains whose
// intermediate tokens were pruned survive to the traceback.  Layer 0 is the start state's closure (cost 0, cutoff beam),
// pruned like every frame; layer t + 1 follows frame t.
#include <cmath>

#include "common.cuh"

namespace ccb {

namespace {

constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
constexpr unsigned kNoArc = 0xFFFFFFFFu;   // the arc id of the start state's token in layer 0
constexpr unsigned long long kEmpty = ~0ull;

__host__ __device__ __forceinline__ size_t Up256(size_t x) { return (x + 255) & ~(size_t)255; }

// Per-utterance workspace: two hash tables (the current and the previous layer), each with the list of its used slots;
// the pruning keys; the kept tokens of both layers; the records of every layer.
struct WsLayout {
    size_t MS = 0, HC = 0, K = 0, R = 0, layers = 0;
    size_t state[2], key[2], tok[2], list[2], sel, kst[2], kco[2], fr_prev, fr_arcs, total;
};

__host__ __device__ inline WsLayout MakeLayout(int S, int L, int E, int D, int T, int K) {
    WsLayout w;
    // distinct states of one layer: the emitting candidates' destinations, each with at most E more through epsilon arcs
    // (layer 0: the start state's closure); never more than the graph has
    const size_t per = (size_t)(E + 1);
    size_t ms = (size_t)K * (size_t)(D > 0 ? D : 1) * per;
    if (ms < per) ms = per;
    w.MS = ms < (size_t)S ? ms : (size_t)S;
    size_t hc = 1;
    while (hc < w.MS + w.MS / 4 + 1) hc <<= 1;
    w.HC = hc;
    w.K = (size_t)K;
    w.R = (size_t)L + 1;
    w.layers = (size_t)T + 1;
    size_t o = 0;
    for (int i = 0; i < 2; ++i) {
        w.state[i] = o; o += Up256(w.HC * 4);
        w.key[i] = o;   o += Up256(w.HC * 8);
        w.tok[i] = o;   o += Up256(w.HC * 4);
        w.list[i] = o;  o += Up256(w.MS * 4);
        w.kst[i] = o;   o += Up256(w.K * 4);
        w.kco[i] = o;   o += Up256(w.K * 4);
    }
    w.sel = o;     o += Up256(w.MS * 8);
    w.fr_prev = o; o += Up256(w.layers * w.K * 4);
    w.fr_arcs = o; o += Up256(w.layers * w.K * w.R * 4);
    w.total = o;
    return w;
}

// float -> u32, monotone (c is never NaN here; -0 is folded into +0 so that the order is the order of the values)
__device__ __forceinline__ unsigned OrderedBits(float c) {
    const unsigned b = __float_as_uint(__fadd_rn(c, 0.f));
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float CostOf(unsigned long long key) {
    const unsigned u = (unsigned)(key >> 32);
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}
__device__ __forceinline__ unsigned long long Key(float c, unsigned id) {
    return ((unsigned long long)OrderedBits(c) << 32) | id;
}

struct Hash {
    int *state;                // -1: empty
    unsigned long long *key;   // (ordered cost bits, file arc id), kEmpty when unset
    int *tok;                  // the kept token's index in its layer (set for kept tokens only)
    int *list;                 // used slots, in insertion order
};

__device__ __forceinline__ unsigned HashOf(int s, unsigned mask) {
    unsigned x = (unsigned)s * 0x9E3779B1u;
    return (x ^ (x >> 15)) & mask;
}

__device__ __forceinline__ void Insert(const Hash &h, unsigned mask, int s, unsigned long long key, int *count) {
    unsigned i = HashOf(s, mask);
    for (;;) {
        const int old = atomicCAS(&h.state[i], -1, s);
        if (old == -1) { h.list[atomicAdd(count, 1)] = (int)i; break; }
        if (old == s) break;
        i = (i + 1) & mask;
    }
    atomicMin(&h.key[i], key);
}

__device__ __forceinline__ int Find(const Hash &h, unsigned mask, int s) {
    unsigned i = HashOf(s, mask);
    while (h.state[i] != s) i = (i + 1) & mask;
    return (int)i;
}

struct Params {
    WfstDev g;
    const void *y;
    int y_dtype;
    int N, T, V, K, wcap;
    const int *len;
    float nacs, wps, beam;
    double acwt, lmwt, wip;
    char *ws;
    WsLayout lay;
    int *words, *num_words, *align, *reached_final;
    float *ac_logp, *graph_cost, *cost;
};

__device__ float BlockMin(float v, float *red) {
    for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    if (warp == 0) {
        v = lane < kWarps ? red[lane] : INFINITY;
        for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
        if (lane == 0) red[0] = v;
    }
    __syncthreads();
    return red[0];
}

__global__ void __launch_bounds__(kThreads) wfst_decode_kernel(const Params P) {
    extern __shared__ float yrow[];
    __shared__ int s_count, s_kept, s_want, s_used[2];
    __shared__ unsigned s_hist[256];
    __shared__ unsigned long long s_prefix, s_best_fin, s_best_any;
    __shared__ float s_red[32];
    const int n = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const WfstDev &g = P.g;
    const WsLayout &W = P.lay;
    const int K = P.K, R = (int)W.R, T = P.T;
    char *base = P.ws + (size_t)n * W.total;
    Hash H[2];
    int *kst[2];
    float *kco[2];
    for (int i = 0; i < 2; ++i) {
        H[i].state = reinterpret_cast<int *>(base + W.state[i]);
        H[i].key = reinterpret_cast<unsigned long long *>(base + W.key[i]);
        H[i].tok = reinterpret_cast<int *>(base + W.tok[i]);
        H[i].list = reinterpret_cast<int *>(base + W.list[i]);
        kst[i] = reinterpret_cast<int *>(base + W.kst[i]);
        kco[i] = reinterpret_cast<float *>(base + W.kco[i]);
    }
    unsigned long long *sel = reinterpret_cast<unsigned long long *>(base + W.sel);
    int *fr_prev = reinterpret_cast<int *>(base + W.fr_prev);
    int *fr_arcs = reinterpret_cast<int *>(base + W.fr_arcs);
    const unsigned mask = (unsigned)(W.HC - 1);
    const int ln = P.len[n];
    int *align = P.align + (size_t)n * T;
    for (int t = tid; t < T; t += kThreads) align[t] = -1;
    for (size_t i = tid; i < W.HC; i += kThreads) {
        H[0].state[i] = -1; H[0].key[i] = kEmpty;
        H[1].state[i] = -1; H[1].key[i] = kEmpty;
    }
    if (tid == 0) { s_count = 0; s_used[0] = s_used[1] = 0; }
    __syncthreads();

    // steps 3 and 4 on the layer in H[c] (its states are in H[c].list[0 .. s_count)): epsilon closure within `cutoff`,
    // then the kept tokens of layer f and their records (the predecessor's index is read from H[c ^ 1])
    auto close_and_prune = [&](int c, float cutoff, int f) {
        const Hash &h = H[c];
        for (int lv = 0; lv <= g.L; ++lv) {
            const int cnt = s_count;
            __syncthreads();
            for (int i = tid; i < cnt; i += kThreads) {
                const int slot = h.list[i], s = h.state[slot];
                const int e0 = g.eps_off[s], e1 = g.arc_off[s + 1];
                if (e0 == e1 || g.level[s] != lv) continue;
                const float cs = CostOf(h.key[slot]);
                for (int j = e0; j < e1; ++j) {
                    float x = __fadd_rn(cs, g.w[j]);
                    if (g.olabel[j] != 0) x = __fadd_rn(x, P.wps);
                    if (x <= cutoff && x < INFINITY) Insert(h, mask, g.dst[j], Key(x, (unsigned)g.fid[j]), &s_count);
                }
            }
            __syncthreads();
        }
        const int cnt = s_count;
        unsigned long long kth = kEmpty;
        if (cnt > K) {
            // radix select of the K-th smallest (ordered cost bits, state): keys are distinct, so exactly K are <= it
            for (int i = tid; i < cnt; i += kThreads) {
                const int slot = h.list[i];
                sel[i] = (h.key[slot] & 0xFFFFFFFF00000000ull) | (unsigned)h.state[slot];
            }
            unsigned long long prefix = 0, pmask = 0;
            int want = K;
            for (int shift = 56; shift >= 0; shift -= 8) {
                for (int i = tid; i < 256; i += kThreads) s_hist[i] = 0;
                __syncthreads();
                for (int i = tid; i < cnt; i += kThreads) {
                    const unsigned long long v = sel[i];
                    if ((v & pmask) == prefix) atomicAdd(&s_hist[(v >> shift) & 255], 1u);
                }
                __syncthreads();
                if (warp == 0) {
                    unsigned loc = 0;
                    for (int b = 0; b < 8; ++b) loc += s_hist[lane * 8 + b];
                    unsigned inc = loc;
                    for (int o = 1; o < 32; o <<= 1) {
                        const unsigned u = __shfl_up_sync(0xffffffffu, inc, o);
                        if (lane >= o) inc += u;
                    }
                    const unsigned exc = inc - loc;
                    const unsigned hit = __ballot_sync(0xffffffffu, exc < (unsigned)want && (unsigned)want <= inc);
                    if (lane == __ffs(hit) - 1) {
                        unsigned cum = exc;
                        for (int b = 0; b < 8; ++b) {
                            const unsigned hb = s_hist[lane * 8 + b];
                            if (cum + hb >= (unsigned)want) {
                                s_prefix = prefix | ((unsigned long long)(lane * 8 + b) << shift);
                                s_want = want - (int)cum;
                                break;
                            }
                            cum += hb;
                        }
                    }
                }
                __syncthreads();
                prefix = s_prefix;
                want = s_want;
                pmask |= 0xFFull << shift;
            }
            kth = prefix;
        }
        if (tid == 0) s_kept = 0;
        __syncthreads();
        const Hash &hp = H[c ^ 1];
        int *pst = fr_prev + (size_t)f * K;
        int *arcs = fr_arcs + (size_t)f * K * R;
        for (int i = tid; i < cnt; i += kThreads) {
            const int slot = h.list[i];
            const int s = h.state[slot];
            if (cnt > K && ((h.key[slot] & 0xFFFFFFFF00000000ull) | (unsigned)s) > kth) continue;
            const int k = atomicAdd(&s_kept, 1);
            kst[c][k] = s;
            kco[c][k] = CostOf(h.key[slot]);
            h.tok[slot] = k;
            // the record: arcs from this token back to the emitting arc of this frame (or to the start state in layer 0)
            int j = 0, prev = -1, sl = slot;
            for (;;) {
                const unsigned id = (unsigned)(h.key[sl] & 0xFFFFFFFFull);
                if (id == kNoArc) break;
                arcs[(size_t)k * R + j++] = (int)id;
                const int a = g.lay[id];
                if (g.tok[a] < 0) { sl = Find(h, mask, g.src[a]); continue; }
                prev = hp.tok[Find(hp, mask, g.src[a])];
                break;
            }
            for (; j < R; ++j) arcs[(size_t)k * R + j] = -1;
            pst[k] = prev;
        }
        __syncthreads();
    };

    int cur = 0;
    if (tid == 0) Insert(H[0], mask, g.start, Key(0.f, kNoArc), &s_count);
    __syncthreads();
    close_and_prune(0, P.beam, 0);
    int nk = s_kept;
    bool dead = false;
    for (int t = 0; t < ln; ++t) {
        const int pv = cur;
        cur ^= 1;
        // clear the hash of two layers ago through its list of used slots
        const Hash &h = H[cur];
        const int used = s_used[cur];
        for (int i = tid; i < used; i += kThreads) { const int sl = h.list[i]; h.state[sl] = -1; h.key[sl] = kEmpty; }
        const size_t yb = ((size_t)n * T + t) * P.V;
        for (int c = tid; c < P.V; c += kThreads) yrow[c] = load_y(P.y, P.y_dtype, (long)(yb + c));
        if (tid == 0) { s_used[pv] = s_count; s_count = 0; }
        __syncthreads();
        // 1. best_e over every emitting candidate (a warp per kept token)
        float best = INFINITY;
        for (int k = warp; k < nk; k += kWarps) {
            const int s = kst[pv][k];
            const float c = kco[pv][k];
            for (int j = g.arc_off[s] + lane; j < g.eps_off[s]; j += 32) {
                float x = __fadd_rn(__fadd_rn(c, g.w[j]), __fmul_rn(P.nacs, yrow[g.tok[j]]));
                if (g.olabel[j] != 0) x = __fadd_rn(x, P.wps);
                best = fminf(best, x);
            }
        }
        const float best_e = BlockMin(best, s_red);
        if (!(best_e < INFINITY)) { dead = true; break; }
        const float cutoff = __fadd_rn(best_e, P.beam);
        // 2. recombination of the candidates within the cutoff
        for (int k = warp; k < nk; k += kWarps) {
            const int s = kst[pv][k];
            const float c = kco[pv][k];
            for (int j = g.arc_off[s] + lane; j < g.eps_off[s]; j += 32) {
                float x = __fadd_rn(__fadd_rn(c, g.w[j]), __fmul_rn(P.nacs, yrow[g.tok[j]]));
                if (g.olabel[j] != 0) x = __fadd_rn(x, P.wps);
                if (x <= cutoff && x < INFINITY) Insert(h, mask, g.dst[j], Key(x, (unsigned)g.fid[j]), &s_count);
            }
        }
        __syncthreads();
        close_and_prune(cur, cutoff, t + 1);
        nk = s_kept;
    }

    // the result: the kept token with the smallest (cost + final, state); without a final state, the smallest (cost, state)
    int *wrow = P.words + (size_t)n * P.wcap;
    if (dead) {
        for (int i = tid; i < P.wcap; i += kThreads) wrow[i] = -1;
        for (int t = tid; t < T; t += kThreads) align[t] = -1;
        if (tid == 0) {
            P.num_words[n] = -1; P.reached_final[n] = 0;
            P.ac_logp[n] = -INFINITY; P.graph_cost[n] = INFINITY; P.cost[n] = INFINITY;
        }
        return;
    }
    if (tid == 0) { s_best_fin = kEmpty; s_best_any = kEmpty; }
    __syncthreads();
    for (int k = tid; k < nk; k += kThreads) {
        const int s = kst[cur][k];
        const float c = kco[cur][k], fin = g.final_cost[s];
        atomicMin(&s_best_any, Key(c, (unsigned)s));
        if (fin < INFINITY) {
            const float fc = __fadd_rn(c, fin);
            if (fc < INFINITY) atomicMin(&s_best_fin, Key(fc, (unsigned)s));
        }
    }
    __syncthreads();
    if (tid == 0) {
        const bool fin = s_best_fin != kEmpty;
        const int s = (int)((fin ? s_best_fin : s_best_any) & 0xFFFFFFFFull);
        int k = H[cur].tok[Find(H[cur], mask, s)];
        double gsum = fin ? (double)g.final_cost[s] : 0.0, asum = 0.0;
        int nw = 0;
        // the path backwards, layer by layer; each record lists its arcs backwards
        for (int f = ln, kk = k; f >= 0; --f) {
            const int *arcs = fr_arcs + ((size_t)f * K + kk) * R;
            for (int j = 0; j < R && arcs[j] >= 0; ++j) {
                const int a = g.lay[arcs[j]];
                gsum += (double)g.w[a];
                if (g.olabel[a] != 0) ++nw;
                if (g.tok[a] >= 0) {
                    align[f - 1] = g.tok[a];
                    asum += (double)load_y(P.y, P.y_dtype, (long)(((size_t)n * T + f - 1) * P.V + g.tok[a]));
                }
            }
            kk = fr_prev[(size_t)f * K + kk];
        }
        int pos = nw;
        for (int f = ln, kk = k; f >= 0; --f) {
            const int *arcs = fr_arcs + ((size_t)f * K + kk) * R;
            for (int j = 0; j < R && arcs[j] >= 0; ++j) {
                const int a = g.lay[arcs[j]];
                if (g.olabel[a] != 0) wrow[--pos] = g.olabel[a];
            }
            kk = fr_prev[(size_t)f * K + kk];
        }
        P.num_words[n] = nw;
        P.reached_final[n] = fin ? 1 : 0;
        P.ac_logp[n] = (float)asum;
        P.graph_cost[n] = (float)gsum;
        P.cost[n] = (float)(P.lmwt * gsum - P.acwt * asum + P.wip * (double)nw);
        s_want = nw;
    }
    __syncthreads();
    for (int i = s_want + tid; i < P.wcap; i += kThreads) wrow[i] = -1;
}

}  // namespace

size_t WfstWsBytes(const WfstDev &g, int N, int T, int K) {
    return (size_t)N * MakeLayout(g.S, g.L, g.E, g.max_out, T, K).total;
}

int LaunchWfstDecode(const WfstDev &g, const void *y, int y_dtype, int N, int T, int V, const int *len, float acwt, float lmwt,
                     float wip, float beam, int K, void *ws, int *words, int *num_words, int *align, float *ac_logp,
                     float *graph_cost, float *cost, int *reached_final, cudaStream_t stream) {
    Params p;
    p.g = g;
    p.y = y; p.y_dtype = y_dtype; p.N = N; p.T = T; p.V = V; p.K = K; p.len = len;
    p.wcap = (T + 1) * (1 + g.L);
    // acs = acwt / lmwt and wps = wip / lmwt in fp32, as the restatement computes them
    p.nacs = -(acwt / lmwt);
    p.wps = wip / lmwt;
    p.beam = beam;
    p.acwt = acwt; p.lmwt = lmwt; p.wip = wip;
    p.ws = reinterpret_cast<char *>(ws);
    p.lay = MakeLayout(g.S, g.L, g.E, g.max_out, T, K);
    p.words = words; p.num_words = num_words; p.align = align; p.reached_final = reached_final;
    p.ac_logp = ac_logp; p.graph_cost = graph_cost; p.cost = cost;
    wfst_decode_kernel<<<N, kThreads, (size_t)V * sizeof(float), stream>>>(p);
    CountLaunch();
    return (int)cudaGetLastError();
}

}  // namespace ccb
