// Transducer (RNN-T, monotonic) beam search: one launch per frame, one CTA per utterance (DESIGN.md §7 "Transducer beam
// search").  The caller runs the predictor and joiner networks between launches; each step reads the (N*B, V) row block of
// the current beam slots and
//   1. selects the B best candidates (r, k), value s_r + lp_r[k] in fp64, by (value desc, flat index r*V + k asc), exactly:
//      the flat index range is scanned in windows, a candidate is kept only when it ranks before the B-th best so far, and
//      the kept ones are bitonic-sorted together with the best B when the buffer fills (or at the end);
//   2. finds the target prefix of each: the slot's own trie node for blank, else the child (node, k), looked up in the
//      utterance's open-addressing hash and created (ids in visiting order) if missing;
//   3. merges candidates with the same target in increasing flat index, logaddexp in fp64, in that order -- no atomics;
//   4. writes each slot of the next beam (order of first appearance): parent slot, token (-1: stay), trie node, score.
// The finish launch ranks the beam by score (stable), walks the trie back and writes the N-best.
// The FUSE instantiation adds an external LM and/or an ILM estimate (DESIGN.md §7 "RNN-T beam search with LM fusion"):
// each slot also carries an LM part lm_r (fp64, caller-owned), a candidate ranks by ((s_r + v) + lm_r) + term, and a new
// slot keeps the LM part of its first candidate while only the acoustic parts s_r + v are merged.  The instantiation
// without it is the plain search.  ngram_slot_rows_kernel produces the n-gram LM's rows for the fused step, and
// lm_mix_slot_rows_kernel the rows of a weighted mix of n-gram and neural LMs.
#include "ngram.h"
#include "transducer_beam.cuh"

namespace ccb {

namespace {

constexpr int kThreads = 512;
constexpr int kSort = 2048;                  // sort buffer: the best B, then the candidates waiting to be sorted
constexpr int kWindow = 2 * kThreads;        // flat indices scanned between two looks at the buffer
constexpr int kNoKey = 0x7fffffff;

__global__ void __launch_bounds__(kThreads) rnnt_beam_init_kernel(int T, int B, char *ws, int *parent, int *token, int *node,
                                                                  double *score) {
    const int n = blockIdx.x;
    const Trie tr = UttTrie(ws, n, T, B);
    for (size_t i = threadIdx.x; i < tr.hslots; i += blockDim.x) tr.hash[i] = -1;
    for (int q = threadIdx.x; q < B; q += blockDim.x) {
        const size_t s = (size_t)n * B + q;
        parent[s] = q; token[s] = -1;
        node[s] = q == 0 ? 0 : -1;
        score[s] = q == 0 ? 0.0 : kNegInf;
    }
    if (threadIdx.x == 0) { tr.parent[0] = -1; tr.tok[0] = -1; *tr.next = 1; }
}

// the fusion inputs of the FUSE instantiation; a null row block turns its term off
struct FuseParams {
    const void *lm_rows;     // (N*B, V) external LM log-probs, or null
    const void *ilm_rows;    // (N*B, V) ILM logits, or null
    int lm_dtype, ilm_dtype;
    double alpha, beta, w;
    double *lm_part;         // (N, B): read for the current beam, written for the next
};

// What extension (r, k), k != blank, adds to the LM part: (beta + alpha LM[k]) + w (I[k] - lse_I), each product and sum
// rounded on its own (no contraction), so that an fp64 restatement reproduces it; -inf when either row entry is -inf.
__device__ __forceinline__ double FuseTerm(const FuseParams &F, long row, int k, float ilse) {
    double term = 0.0;
    if (F.lm_rows) {
        const float lm = load_y(F.lm_rows, F.lm_dtype, row + k);
        if (lm == -INFINITY) return kNegInf;
        term = __dadd_rn(F.beta, __dmul_rn(F.alpha, (double)lm));
    }
    if (F.ilm_rows) {
        const float z = load_y(F.ilm_rows, F.ilm_dtype, row + k);
        if (z == -INFINITY) return kNegInf;
        const float x = z - ilse;
        term = F.lm_rows ? __dadd_rn(term, __dmul_rn(F.w, (double)x)) : __dmul_rn(F.w, (double)x);
    }
    return term;
}

template <bool FUSE>
__global__ void __launch_bounds__(kThreads) rnnt_beam_step_kernel(const StepParams P, const FuseParams F) {
    __shared__ double sort_m[kSort];
    __shared__ int sort_k[kSort];
    __shared__ double s_score[kBeamMax], o_m[kBeamMax];
    __shared__ int s_node[kBeamMax], o_f[kBeamMax], o_tgt[kBeamMax], o_first[kBeamMax];
    __shared__ float s_lse[kBeamMax];
    __shared__ double s_lm[FUSE ? kBeamMax : 1];      // FUSE: the slots' LM parts
    __shared__ float s_ilse[FUSE ? kBeamMax : 1];     // FUSE: the ILM rows' normalisers over the non-blank columns
    __shared__ int s_nb, s_cnt, s_kept;
    const int n = blockIdx.x, tid = threadIdx.x;
    const int B = P.B, V = P.V, T = P.T, t = P.t;
    const size_t slot0 = (size_t)n * B;
    if (t >= P.len[n]) {   // the utterance has ended: every slot stays itself
        for (int q = tid; q < B; q += blockDim.x) { P.parent[slot0 + q] = q; P.token[slot0 + q] = -1; }
        return;
    }
    for (int q = tid; q < B; q += blockDim.x) { s_score[q] = P.score[slot0 + q]; s_node[q] = P.node[slot0 + q]; }
    if constexpr (FUSE)
        for (int q = tid; q < B; q += blockDim.x) s_lm[q] = F.lm_part[slot0 + q];
    for (int i = tid; i < B; i += blockDim.x) { sort_m[i] = kNegInf; sort_k[i] = kNoKey; }
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    if (tid == 0) {   // the live slots are a prefix of the beam
        int nb = 0;
        while (nb < B && s_score[nb] > kNegInf) ++nb;
        s_nb = nb;
    }
    __syncthreads();
    const int nb = s_nb;
    const long frow = ((long)n * T + t) * V;
    // row normalisers (modes 1, 2): one warp per row, an online (max, sum of exp) in fp32, merged in a fixed tree
    if (P.mode != 0) {
        const int lane = tid & 31, warp = tid >> 5;
        for (int r = warp; r < nb; r += blockDim.x >> 5) {
            const long row = (long)(slot0 + r) * V;
            float m = -INFINITY, s = 0.f;
            for (int k = lane; k < V; k += 32) {
                const float z = RowZ(P, row, frow, k);
                if (z == -INFINITY) continue;
                if (z > m) { s = s * expf(m - z) + 1.f; m = z; } else { s += expf(z - m); }
            }
            for (int o = 16; o > 0; o >>= 1) {
                const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
                const float mm = fmaxf(m, m2);
                if (mm > -INFINITY) s = (m > -INFINITY ? s * expf(m - mm) : 0.f) + (m2 > -INFINITY ? s2 * expf(m2 - mm) : 0.f);
                m = mm;
            }
            if (lane == 0) s_lse[r] = m > -INFINITY ? m + logf(s) : -INFINITY;
        }
        __syncthreads();
    }
    // FUSE: the ILM rows' normalisers, the same online (max, sum of exp) over the non-blank columns (written out again:
    // a shared inline function changes the unfused step's register allocation)
    if constexpr (FUSE) {
        if (F.ilm_rows) {
            const int lane = tid & 31, warp = tid >> 5;
            for (int r = warp; r < nb; r += blockDim.x >> 5) {
                const long row = (long)(slot0 + r) * V;
                float m = -INFINITY, s = 0.f;
                for (int k = lane; k < V; k += 32) {
                    const float z = k == P.blank ? -INFINITY : load_y(F.ilm_rows, F.ilm_dtype, row + k);
                    if (z == -INFINITY) continue;
                    if (z > m) { s = s * expf(m - z) + 1.f; m = z; } else { s += expf(z - m); }
                }
                for (int o = 16; o > 0; o >>= 1) {
                    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
                    const float mm = fmaxf(m, m2);
                    if (mm > -INFINITY)
                        s = (m > -INFINITY ? s * expf(m - mm) : 0.f) + (m2 > -INFINITY ? s2 * expf(m2 - mm) : 0.f);
                    m = mm;
                }
                if (lane == 0) s_ilse[r] = m > -INFINITY ? m + logf(s) : -INFINITY;
            }
            __syncthreads();
        }
    }
    // 1. exact top-B over the nb * V candidates
    const int total = nb * V;
    const int cap = kSort - B;
    for (int w0 = 0; w0 < total; w0 += kWindow) {
        const double thr_m = sort_m[B - 1];
        const int thr_k = sort_k[B - 1];
        for (int f = w0 + tid; f < min(total, w0 + kWindow); f += blockDim.x) {
            const int r = f / V, k = f - r * V;
            const long row = (long)(slot0 + r) * V;
            float v = RowZ(P, row, frow, k);
            if (P.mode != 0) v = v - s_lse[r];
            double m = s_score[r] + (double)v;
            if constexpr (FUSE) {
                m = m + s_lm[r];
                if (k != P.blank) {
                    const double term = FuseTerm(F, row, k, F.ilm_rows ? s_ilse[r] : 0.f);
                    m = term == kNegInf ? kNegInf : m + term;
                }
            }
            if (m > kNegInf && Before(m, f, thr_m, thr_k)) {
                const int pos = atomicAdd(&s_cnt, 1);
                sort_m[B + pos] = m;
                sort_k[B + pos] = f;
            }
        }
        __syncthreads();
        const int cnt = s_cnt;
        if (cnt > 0 && (cnt > cap - kWindow || w0 + kWindow >= total)) {
            const int ps = Pow2Ceil(B + cnt);
            for (int i = B + cnt + tid; i < ps; i += blockDim.x) { sort_m[i] = kNegInf; sort_k[i] = kNoKey; }
            __syncthreads();
            BitonicSort(sort_m, sort_k, ps);
            if (tid == 0) s_cnt = 0;
        }
        __syncthreads();
    }
    if (tid == 0) {
        int k = 0;
        while (k < B && sort_m[k] > kNegInf) ++k;
        s_kept = k;
    }
    __syncthreads();
    const int kept = s_kept;
    // 2. the kept candidates in visiting order (increasing flat index) and their target trie nodes
    for (int j = tid; j < kept; j += blockDim.x) {
        int pos = 0;
        for (int i = 0; i < kept; ++i) pos += sort_k[i] < sort_k[j];
        o_f[pos] = sort_k[j];
        o_m[pos] = sort_m[j];
    }
    __syncthreads();
    const Trie tr = UttTrie(P.ws, n, T, B);
    for (int j = tid; j < kept; j += blockDim.x) {
        const int r = o_f[j] / V, k = o_f[j] - r * V, parent = s_node[r];
        int found = -1;
        if (k == P.blank) {
            found = parent;
        } else {
            for (unsigned h = TrieHash(parent, k, tr.hslots);; h = (h + 1) & (unsigned)(tr.hslots - 1)) {
                const int x = tr.hash[h];
                if (x < 0) break;
                if (tr.parent[x] == parent && tr.tok[x] == k) { found = x; break; }
            }
        }
        o_tgt[j] = found;
    }
    __syncthreads();
    if (tid == 0) {   // missing children created in visiting order (distinct: the beam's prefixes are distinct)
        int next = *tr.next;
        for (int j = 0; j < kept; ++j) {
            if (o_tgt[j] >= 0) continue;
            const int r = o_f[j] / V, k = o_f[j] - r * V, x = next++;
            tr.parent[x] = s_node[r]; tr.tok[x] = k;
            unsigned h = TrieHash(s_node[r], k, tr.hslots);
            while (tr.hash[h] >= 0) h = (h + 1) & (unsigned)(tr.hslots - 1);
            tr.hash[h] = x;
            o_tgt[j] = x;
        }
        *tr.next = next;
    }
    __syncthreads();
    // 3. the first candidate of each target and its position in the next beam
    for (int j = tid; j < kept; j += blockDim.x) {
        int first = j;
        for (int i = 0; i < j; ++i)
            if (o_tgt[i] == o_tgt[j]) { first = i; break; }
        o_first[j] = first;
    }
    __syncthreads();
    // 4. the next beam: slot q from its first candidate j, the later ones with the same target folded in visiting order
    for (int j = tid; j < kept; j += blockDim.x) {
        if (o_first[j] != j) continue;
        int q = 0;
        for (int i = 0; i < j; ++i) q += o_first[i] == i;
        if constexpr (FUSE) {
            const int r = o_f[j] / V, k = o_f[j] - r * V;
            // only the acoustic parts s_r + v are merged (recomputed from the rows); the slot keeps its first candidate's
            // LM part
            auto acoustic = [&](int f) {
                const int r2 = f / V, k2 = f - r2 * V;
                float v = RowZ(P, (long)(slot0 + r2) * V, frow, k2);
                if (P.mode != 0) v = v - s_lse[r2];
                return s_score[r2] + (double)v;
            };
            double s = acoustic(o_f[j]);
            for (int i = j + 1; i < kept; ++i)
                if (o_tgt[i] == o_tgt[j]) s = lse(s, acoustic(o_f[i]));
            P.parent[slot0 + q] = r;
            P.token[slot0 + q] = k == P.blank ? -1 : k;
            P.node[slot0 + q] = o_tgt[j];
            P.score[slot0 + q] = s;
            F.lm_part[slot0 + q] = k == P.blank ? s_lm[r]
                                                : s_lm[r] + FuseTerm(F, (long)(slot0 + r) * V, k, F.ilm_rows ? s_ilse[r] : 0.f);
        } else {
            double s = o_m[j];
            for (int i = j + 1; i < kept; ++i)
                if (o_tgt[i] == o_tgt[j]) s = lse(s, o_m[i]);
            const int r = o_f[j] / V, k = o_f[j] - r * V;
            P.parent[slot0 + q] = r;
            P.token[slot0 + q] = k == P.blank ? -1 : k;
            P.node[slot0 + q] = o_tgt[j];
            P.score[slot0 + q] = s;
        }
    }
    if (tid == 0) {
        int nb2 = 0;
        for (int j = 0; j < kept; ++j) nb2 += o_first[j] == j;
        s_cnt = nb2;
    }
    __syncthreads();
    for (int q = s_cnt + tid; q < B; q += blockDim.x) {
        P.parent[slot0 + q] = q; P.token[slot0 + q] = -1; P.node[slot0 + q] = -1; P.score[slot0 + q] = kNegInf;
        if constexpr (FUSE) F.lm_part[slot0 + q] = 0.0;
    }
}

constexpr int kRowThreads = 256;
constexpr int kChainMax = kNgramMaxOrder + 1;   // a state of order k backs off to the root in k - 1 steps

// One CTA per slot q of the next beam: its LM state (its parent's, advanced by its token when it emitted one; every slot
// at the start state, after </s>, when parent is null) and its dense row ln P(. | state), fp32.  The row is built along the
// back-off chain s_0 = state, s_j = back[s_j-1], ..., root in word space (shared memory, fp64): every word starts at
// C_root + root_p[w], then the arcs of each chain state, from the root's child down to s_0, overwrite their words with
// C_j + p (C_j = bow[s_0] + ... + bow[s_j-1], summed in that order), so that each word holds what LmLog10's walk returns;
// arcs whose probability is NaN (prefixes the loader inserted) back off.  A token without an LM word (the blank label 0)
// gets 0 and keeps the state.
__global__ void __launch_bounds__(kRowThreads) ngram_slot_rows_kernel(const NGramDev lm, int W, int V, int B,
                                                                      const int *parent, const int *token,
                                                                      const int *state_in, int *state_out, float *rows) {
    extern __shared__ double wrow[];   // [W]
    __shared__ int s_chain[kChainMax];
    __shared__ double s_c[kChainMax];
    __shared__ int s_len;
    const int q = blockIdx.x, tid = threadIdx.x;
    if (tid == 0) {
        int s = lm.root_dst[lm.eos];
        if (parent) {
            s = state_in[(size_t)(q / B) * B + parent[q]];
            const int w = token[q] >= 0 ? lm.tok2word[token[q]] : -1;
            if (w >= 0) { int d; LmLog10(lm, s, w, &d); s = d; }
        }
        state_out[q] = s;
        int L = 0;
        double c = 0.0;
        for (;;) {   // the chain ends at the root (state 0)
            s_chain[L] = s; s_c[L] = c;
            if (s == 0) break;
            c += (double)lm.bow[s];
            s = lm.back[s];
            ++L;
        }
        s_len = L;
    }
    __syncthreads();
    const int L = s_len;
    const double croot = s_c[L];
    for (int w = tid; w < W; w += blockDim.x) wrow[w] = croot + (double)lm.root_p[w];
    __syncthreads();
    for (int j = L - 1; j >= 0; --j) {   // the words of one state's arcs are distinct: no two threads write one word
        const int s = s_chain[j];
        const double c = s_c[j];
        for (int a = lm.arc_off[s] + tid; a < lm.arc_off[s + 1]; a += blockDim.x) {
            const float p = lm.arc_p[a];
            if (p == p) wrow[lm.arc_word[a]] = c + (double)p;
        }
        __syncthreads();
    }
    float *out = rows + (size_t)q * V;
    for (int k = tid; k < V; k += blockDim.x) {
        const int w = lm.tok2word[k];
        out[k] = w < 0 ? 0.f : (float)__dmul_rn(wrow[w], kLn10);
    }
}

// acc after a member's value v of weight w: the product rounded on its own, then the sum (the first product starts it);
// a -inf value, and a -inf sum, stay -inf
__device__ __forceinline__ void MixAdd(double &acc, bool first, double w, float v) {
    if (v == -INFINITY || (!first && acc == kNegInf)) { acc = kNegInf; return; }
    const double x = __dmul_rn(w, (double)v);
    acc = first ? x : __dadd_rn(acc, x);
}

// One CTA per slot q of the next beam: the mix row MIX[k] = sum_i w_i LM_i[k] of an LM mix (DESIGN.md §7 "RNN-T beam search
// with an LM mix"), fp32.  Members are visited in the mix's order.  An n-gram member advances its state and builds its word
// row exactly as ngram_slot_rows_kernel does (the shared word row is rebuilt per member), and contributes the fp32 value
// that kernel writes; a neural member contributes its row block's entry, widened exactly.  Each product w_i LM_i[k] and
// each sum is rounded in fp64 on its own, the first product starting the sum; a -inf in any member makes the entry -inf.
// Each thread owns the labels k = tid (mod blockDim) of the fp64 accumulator for the whole launch.
__global__ void __launch_bounds__(kRowThreads) lm_mix_slot_rows_kernel(const LmMixDev mix, int V, int B, const int *parent,
                                                                       const int *token, float *rows) {
    extern __shared__ double smem[];   // [V] label accumulator, then [W] word row
    double *acc = smem, *wrow = smem + V;
    __shared__ int s_chain[kChainMax];
    __shared__ double s_c[kChainMax];
    __shared__ int s_len;
    const int q = blockIdx.x, tid = threadIdx.x;
    const size_t row = (size_t)q * V;
    for (int i = 0; i < mix.K; ++i) {
        const LmMixMember &m = mix.m[i];
        if (m.rows) {   // a neural member's row block
            for (int k = tid; k < V; k += blockDim.x) MixAdd(acc[k], i == 0, m.w, load_y(m.rows, m.dtype, (long)(row + k)));
            continue;
        }
        const NGramDev &lm = m.lm;
        if (tid == 0) {
            int s = lm.root_dst[lm.eos];
            if (parent) {
                s = m.state_in[(size_t)(q / B) * B + parent[q]];
                const int w = token[q] >= 0 ? lm.tok2word[token[q]] : -1;
                if (w >= 0) { int d; LmLog10(lm, s, w, &d); s = d; }
            }
            m.state_out[q] = s;
            int L = 0;
            double c = 0.0;
            for (;;) {
                s_chain[L] = s; s_c[L] = c;
                if (s == 0) break;
                c += (double)lm.bow[s];
                s = lm.back[s];
                ++L;
            }
            s_len = L;
        }
        __syncthreads();   // (also: the previous n-gram member's word row has been read)
        const int L = s_len;
        const double croot = s_c[L];
        for (int w = tid; w < m.W; w += blockDim.x) wrow[w] = croot + (double)lm.root_p[w];
        __syncthreads();
        for (int j = L - 1; j >= 0; --j) {
            const int s = s_chain[j];
            const double c = s_c[j];
            for (int a = lm.arc_off[s] + tid; a < lm.arc_off[s + 1]; a += blockDim.x) {
                const float p = lm.arc_p[a];
                if (p == p) wrow[lm.arc_word[a]] = c + (double)p;
            }
            __syncthreads();
        }
        for (int k = tid; k < V; k += blockDim.x) {
            const int w = lm.tok2word[k];
            MixAdd(acc[k], i == 0, m.w, w < 0 ? 0.f : (float)__dmul_rn(wrow[w], kLn10));
        }
        __syncthreads();   // s_len and the word row are rewritten by the next n-gram member
    }
    for (int k = tid; k < V; k += blockDim.x) rows[row + k] = (float)acc[k];
}

// ranks the beam by score (desc; ties: beam order) and writes the first nbest rows: tokens -1 padded, lengths (-1 past the
// hypotheses found), scores (-inf there)
__global__ void __launch_bounds__(kThreads) rnnt_beam_finish_kernel(int T, int B, int nbest, const char *ws, const int *node,
                                                                    const double *score, int *tokens, int *lengths,
                                                                    float *scores) {
    __shared__ double s_score[kBeamMax];
    __shared__ int s_nb;
    const int n = blockIdx.x, tid = threadIdx.x;
    const size_t slot0 = (size_t)n * B;
    for (int q = tid; q < B; q += blockDim.x) s_score[q] = score[slot0 + q];
    __syncthreads();
    if (tid == 0) {
        int nb = 0;
        while (nb < B && s_score[nb] > kNegInf) ++nb;
        s_nb = nb;
    }
    __syncthreads();
    const int nb = s_nb;
    const Trie tr = UttTrie(const_cast<char *>(ws), n, T, B);
    const size_t row0 = (size_t)n * nbest;
    for (int q = tid; q < B; q += blockDim.x) {
        int pos = q, x = -1;
        if (q < nb) {
            pos = 0;
            for (int j = 0; j < nb; ++j) pos += Before(s_score[j], j, s_score[q], q);
            x = node[slot0 + q];
        }
        if (pos >= nbest) continue;
        int *tk = tokens + (row0 + pos) * T;
        int L = -1;
        if (x >= 0) {
            L = 0;
            for (int y = x; y > 0; y = tr.parent[y]) ++L;
            int i = L;
            for (int y = x; y > 0; y = tr.parent[y]) tk[--i] = tr.tok[y];
        }
        for (int i = max(L, 0); i < T; ++i) tk[i] = -1;
        lengths[row0 + pos] = L;
        scores[row0 + pos] = x >= 0 ? (float)s_score[q] : -INFINITY;
    }
}

}  // namespace

size_t RnntBeamWsBytes(int N, int T, int B) { return (size_t)N * UttBytes(T, B); }

int LaunchRnntBeamInit(int N, int T, int B, void *ws, int *parent, int *token, int *node, double *score, cudaStream_t s) {
    rnnt_beam_init_kernel<<<N, kThreads, 0, s>>>(T, B, reinterpret_cast<char *>(ws), parent, token, node, score);
    CountLaunch();
    return (int)cudaGetLastError();
}

int LaunchRnntBeamStep(const void *rows, const void *enc, int dtype, int mode, int N, int T, int B, int V, int t,
                       const int *len, int blank, void *ws, int *parent, int *token, int *node, double *score, cudaStream_t s) {
    StepParams p;
    p.rows = rows; p.enc = enc; p.dtype = dtype; p.mode = mode;
    p.N = N; p.T = T; p.B = B; p.V = V; p.t = t; p.blank = blank;
    p.len = len; p.ws = reinterpret_cast<char *>(ws);
    p.parent = parent; p.token = token; p.node = node; p.score = score;
    rnnt_beam_step_kernel<false><<<N, kThreads, 0, s>>>(p, FuseParams{});
    CountLaunch();
    return (int)cudaGetLastError();
}

int LaunchRnntBeamStepFused(const void *rows, const void *enc, int dtype, int mode, int N, int T, int B, int V, int t,
                            const int *len, int blank, void *ws, int *parent, int *token, int *node, double *score,
                            const void *lm_rows, int lm_dtype, double alpha, double beta, const void *ilm_rows, int ilm_dtype,
                            double ilm_weight, double *lm_part, cudaStream_t s) {
    StepParams p;
    p.rows = rows; p.enc = enc; p.dtype = dtype; p.mode = mode;
    p.N = N; p.T = T; p.B = B; p.V = V; p.t = t; p.blank = blank;
    p.len = len; p.ws = reinterpret_cast<char *>(ws);
    p.parent = parent; p.token = token; p.node = node; p.score = score;
    FuseParams f;
    f.lm_rows = lm_rows; f.ilm_rows = ilm_rows; f.lm_dtype = lm_dtype; f.ilm_dtype = ilm_dtype;
    f.alpha = alpha; f.beta = beta; f.w = ilm_weight; f.lm_part = lm_part;
    rnnt_beam_step_kernel<true><<<N, kThreads, 0, s>>>(p, f);
    CountLaunch();
    return (int)cudaGetLastError();
}

size_t NgramSlotRowsSmemBytes(int W) { return (size_t)W * sizeof(double); }

int LaunchNgramSlotRows(const NGramDev &lm, int W, int N, int B, int V, const int *parent, const int *token,
                        const int *state_in, int *state_out, float *rows, cudaStream_t s) {
    const size_t smem = NgramSlotRowsSmemBytes(W);
    if (smem > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute(ngram_slot_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                   (int)smem);
        if (e != cudaSuccess) return (int)e;
    }
    ngram_slot_rows_kernel<<<N * B, kRowThreads, smem, s>>>(lm, W, V, B, parent, token, state_in, state_out, rows);
    CountLaunch();
    return (int)cudaGetLastError();
}

size_t LmMixSlotRowsSmemBytes(int W, int V) { return ((size_t)W + V) * sizeof(double); }

int LaunchLmMixSlotRows(const LmMixDev &mix, int W, int N, int B, int V, const int *parent, const int *token, float *rows,
                        cudaStream_t s) {
    const size_t smem = LmMixSlotRowsSmemBytes(W, V);
    if (smem > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute(lm_mix_slot_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                   (int)smem);
        if (e != cudaSuccess) return (int)e;
    }
    lm_mix_slot_rows_kernel<<<N * B, kRowThreads, smem, s>>>(mix, V, B, parent, token, rows);
    CountLaunch();
    return (int)cudaGetLastError();
}

int LaunchRnntBeamFinish(int N, int T, int B, int nbest, const void *ws, const int *node, const double *score, int *tokens,
                         int *lengths, float *scores, cudaStream_t s) {
    rnnt_beam_finish_kernel<<<N, kThreads, 0, s>>>(T, B, nbest, reinterpret_cast<const char *>(ws), node, score, tokens,
                                                   lengths, scores);
    CountLaunch();
    return (int)cudaGetLastError();
}

}  // namespace ccb
