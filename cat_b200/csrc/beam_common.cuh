// Helpers shared by the prefix searches that keep a per-utterance trie: the CTC prefix beam search (beam_search.cu) and the
// transducer beam search (rnnt_decode.cu).  One CTA per utterance in both; the trie lives in the caller's workspace.  Both
// score a token n-gram LM by the same back-off walk, LmLog10.
#pragma once
#include <cmath>

#include "common.cuh"

namespace ccb {

namespace {

constexpr double kNegInf = -INFINITY;

__host__ __device__ __forceinline__ int Pow2Ceil(int x) {
    int p = 1;
    while (p < x) p <<= 1;
    return p;
}

__host__ __device__ __forceinline__ size_t Up256(size_t x) { return (x + 255) & ~(size_t)255; }

// a trie of T frames with at most B new nodes per frame, plus the root; its hash table at most half full
__host__ __device__ __forceinline__ size_t NodeCap(int T, int B) { return (size_t)B * (size_t)T + 1; }
__host__ __device__ __forceinline__ size_t HashSlots(int T, int B) {
    size_t h = 1;
    while (h < 2 * NodeCap(T, B)) h <<= 1;
    return h;
}

// log(exp(a) + exp(b)) in fp64: the larger plus log1p(exp(smaller - larger)); exact when one side is -inf
__device__ __forceinline__ double lse(double a, double b) {
    const double m = fmax(a, b), o = fmin(a, b);
    if (o == kNegInf) return m;
    return m + log1p(exp(o - m));
}

// a ranks before b: larger mass, then smaller key
__device__ __forceinline__ bool Before(double ma, int ka, double mb, int kb) { return ma > mb || (ma == mb && ka < kb); }

// bitonic sort of m/k[0, P) into Before order (P a power of two), by the whole CTA
__device__ void BitonicSort(double *m, int *k, int P) {
    for (int size = 2; size <= P; size <<= 1)
        for (int j = size >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < P; i += blockDim.x) {
                const int x = i ^ j;
                if (x > i) {
                    const bool up = (i & size) == 0;
                    const bool sw = up ? Before(m[x], k[x], m[i], k[i]) : Before(m[i], k[i], m[x], k[x]);
                    if (sw) {
                        const double tm = m[i]; m[i] = m[x]; m[x] = tm;
                        const int tk = k[i]; k[i] = k[x]; k[x] = tk;
                    }
                }
            }
            __syncthreads();
        }
}

// open-addressing hash of a trie node (parent, token); slots a power of two
__device__ __forceinline__ unsigned TrieHash(int parent, int tok, size_t slots) {
    return (unsigned)((((unsigned)parent * 0x9E3779B1u) ^ ((unsigned)tok * 0x85EBCA77u)) & (unsigned)(slots - 1));
}

constexpr double kLn10 = 2.302585092994045684;

// log10 P(word w | LM state s) by the back-off walk (ngram.h); *dst the state after w.  An arc whose probability is NaN
// was inserted by the loader's prefix closure: it gives the destination, the probability is the back-off value.
__device__ __forceinline__ double LmLog10(const NGramDev &lm, int s, int w, int *dst) {
    double acc = 0.0;
    int d = -1;
    for (;;) {
        if (s == 0) {
            acc += (double)lm.root_p[w];
            if (d < 0) d = lm.root_dst[w];
            break;
        }
        int lo = lm.arc_off[s];
        const int end = lm.arc_off[s + 1];
        int hi = end;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (lm.arc_word[mid] < w) lo = mid + 1; else hi = mid;
        }
        if (lo < end && lm.arc_word[lo] == w) {
            if (d < 0) d = lm.arc_dst[lo];
            const float p = lm.arc_p[lo];
            if (p == p) { acc += (double)p; break; }
        }
        acc += (double)lm.bow[s];
        s = lm.back[s];
    }
    *dst = d;
    return acc;
}

}  // namespace

}  // namespace ccb
