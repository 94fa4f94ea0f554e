// Sentence scores under a token n-gram LM, as CAT's NGram.score computes them for cat.lm.rescore and cat.lm.ppl (DESIGN.md
// §7 "N-gram sentence scoring").  Row b of length L scores the words w_0 .. w_L: w_i is the word of ids[b][i] for i < L
// (token 0 is </s>, and <s> at position 0), w_L the word of the row's last target; the score is ln 10 times the fp64 sum
// of log10 P(w_i | the n-1 words before it), each term LmLog10's back-off walk.
//   Parallel over words: the LM state before w_i is the state the destination rule reaches from the root over the at most
// n-1 preceding words (the rule always reaches the longest suffix of the history that is a state, and no state is longer
// than n-1 words), so every term is computed on its own, without the sequential walk over the row.
//   Deterministic sums: term i goes to slot i mod kSlots, each slot adds its terms in increasing i starting from -0.0 (the
// exact additive identity), and the slots are combined by one fixed binary tree (slot j += slot j + h for h = kSlots/2,
// ..., 1).  Both layouts below evaluate that same tree, so a row's bits depend on the row alone: rows of at most
// kWarpWords words are scored one warp per row, longer ones one CTA of kSlots threads per row; a call picks the layout from
// its width U.
#include "ngram.h"
#include "beam_common.cuh"

namespace ccb {

namespace {

constexpr int kSlots = 1024;                   // the tree's leaves; one thread per slot in the CTA layout
constexpr int kWarpWords = 256;                // the warp layout: lane l holds slots l + 32 k, k < 8
constexpr int kWarpThreads = 256;              // 8 rows per CTA in the warp layout

__device__ __forceinline__ long long LoadInt(const void *p, size_t i, int i64) {
    return i64 ? reinterpret_cast<const long long *>(p)[i] : (long long)reinterpret_cast<const int *>(p)[i];
}

// the row's length, or -1 outside [1, U]
__device__ __forceinline__ int RowLen(const NGramScoreArgs &a, int b) {
    if (!a.lens) return a.U;
    const long long L = LoadInt(a.lens, b, a.lens_i64);
    return L >= 1 && L <= a.U ? (int)L : -1;
}

// the LM word w_i of row b (length L), or -1 for a token outside [0, V)
__device__ __forceinline__ int RowWord(const NGramScoreArgs &a, int b, int L, int i) {
    const long long t = i < L ? LoadInt(a.ids, (size_t)b * a.ids_stride + i, a.ids_i64)
                              : LoadInt(a.last, (size_t)b * a.last_stride, a.last_i64);
    if (t < 0 || t >= a.V) return -1;
    if (t == 0) return i == 0 ? a.bos_word : a.lm.eos;
    return a.lm.tok2word[t];
}

// the state after word w from state s: the destination of the first arc of w on s's back-off chain (root_dst[w] at the
// root), which is the state LmLog10 returns, without its probability walk
__device__ __forceinline__ int LmNext(const NGramDev &lm, int s, int w) {
    for (; s != 0; s = lm.back[s]) {
        int lo = lm.arc_off[s];
        const int end = lm.arc_off[s + 1];
        int hi = end;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (lm.arc_word[mid] < w) lo = mid + 1; else hi = mid;
        }
        if (lo < end && lm.arc_word[lo] == w) return lm.arc_dst[lo];
    }
    return lm.root_dst[w];
}

// log10 P(w_i | w_max(0, i-n+1) .. w_i-1); NaN when one of these words is a bad token
__device__ __forceinline__ double Term(const NGramScoreArgs &a, int b, int L, int i) {
    const int w = RowWord(a, b, L, i);
    if (w < 0) return (double)NAN;
    int s = 0;
    for (int j = max(0, i - a.order + 1); j < i; ++j) {
        const int v = RowWord(a, b, L, j);
        if (v < 0) return (double)NAN;
        s = LmNext(a.lm, s, v);
    }
    int d;
    return LmLog10(a.lm, s, w, &d);
}

// slot i of a row with at most kWarpWords words: its one term, or the identity
__device__ __forceinline__ double Slot(const NGramScoreArgs &a, int b, int L, int i) {
    return i <= L ? Term(a, b, L, i) : -0.0;
}

// the tree's levels h = 16 .. 1 over a warp's 32 slots; lane 0 gets the sum
__device__ __forceinline__ double WarpTree(double x) {
#pragma unroll
    for (int h = 16; h >= 1; h >>= 1) x = __dadd_rn(x, __shfl_down_sync(0xffffffffu, x, h));
    return x;
}

__device__ __forceinline__ float LnScore(double log10_sum) { return (float)__dmul_rn(log10_sum, kLn10); }

// One warp per row, rows of at most kWarpWords words (U < kWarpWords): each slot holds at most one term, slots past
// kWarpWords are the identity, so the tree's levels 512 and 256 are skipped and 128, 64, 32 are done within the lane.
__global__ void __launch_bounds__(kWarpThreads, 4) ngram_score_warp_kernel(const NGramScoreArgs a) {
    const int lane = threadIdx.x & 31;
    const int b = blockIdx.x * (kWarpThreads / 32) + (threadIdx.x >> 5);
    if (b >= a.R) return;
    const int L = RowLen(a, b);
    if (L < 0) {
        if (lane == 0) a.out[b] = NAN;
        return;
    }
    // levels 128 (slot k + 4 into k), 64 (k + 2 into k) and 32, evaluated pair by pair to keep few terms live
    const double s0 = __dadd_rn(Slot(a, b, L, lane), Slot(a, b, L, lane + 128)),
                 s2 = __dadd_rn(Slot(a, b, L, lane + 64), Slot(a, b, L, lane + 192));
    const double s1 = __dadd_rn(Slot(a, b, L, lane + 32), Slot(a, b, L, lane + 160)),
                 s3 = __dadd_rn(Slot(a, b, L, lane + 96), Slot(a, b, L, lane + 224));
    const double s = WarpTree(__dadd_rn(__dadd_rn(s0, s2), __dadd_rn(s1, s3)));
    if (lane == 0) a.out[b] = LnScore(s);
}

// One CTA of kSlots threads per row: thread t is slot t and adds the terms i = t, t + kSlots, ... in that order.
__global__ void __launch_bounds__(kSlots) ngram_score_row_kernel(const NGramScoreArgs a) {
    __shared__ double part[kSlots];
    const int b = blockIdx.x, t = threadIdx.x;
    const int L = RowLen(a, b);
    if (L < 0) {
        if (t == 0) a.out[b] = NAN;
        return;
    }
    double acc = -0.0;
    for (int i = t; i <= L; i += kSlots) acc = __dadd_rn(acc, Term(a, b, L, i));
    part[t] = acc;
    __syncthreads();
    for (int h = kSlots / 2; h >= 32; h >>= 1) {
        if (t < h) part[t] = __dadd_rn(part[t], part[t + h]);
        __syncthreads();
    }
    if (t < 32) {
        const double s = WarpTree(part[t]);
        if (t == 0) a.out[b] = LnScore(s);
    }
}

}  // namespace

int LaunchNgramScore(const NGramScoreArgs &a, cudaStream_t s) {
    if (a.U < kWarpWords)
        ngram_score_warp_kernel<<<(a.R + kWarpThreads / 32 - 1) / (kWarpThreads / 32), kWarpThreads, 0, s>>>(a);
    else
        ngram_score_row_kernel<<<a.R, kSlots, 0, s>>>(a);
    CountLaunch();
    return (int)cudaGetLastError();
}

}  // namespace ccb
