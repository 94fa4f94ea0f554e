// The transducer beam searches' shared pieces: the RNN-T step (rnnt_decode.cu) and the CTC-T step (ctct_decode.cu) keep one
// trie per utterance at the start of the workspace, at the same stride, and read the same row inputs.
#pragma once
#include "beam_common.cuh"
#include "common.cuh"

namespace ccb {

namespace {

// per utterance: parent and token of every node, the hash table (node ids, -1 = empty), the next free node id
__host__ __device__ __forceinline__ size_t UttBytes(int T, int B) {
    return Up256((2 * NodeCap(T, B) + HashSlots(T, B) + 1) * sizeof(int));
}

struct Trie {
    int *parent, *tok, *hash, *next;
    size_t hslots;
};

__device__ __forceinline__ Trie UttTrie(char *ws, int n, int T, int B) {
    Trie tr;
    const size_t cap = NodeCap(T, B);
    tr.parent = reinterpret_cast<int *>(ws + (size_t)n * UttBytes(T, B));
    tr.tok = tr.parent + cap;
    tr.hash = tr.tok + cap;
    tr.hslots = HashSlots(T, B);
    tr.next = tr.hash + tr.hslots;
    return tr;
}

struct StepParams {
    const void *rows;    // (N*B, V): log-probs (mode 0), raw logits (1) or the LogAdd g rows (2)
    const void *enc;     // mode 2: f (N, T, V)
    int dtype, mode;
    int N, T, B, V, t, blank;
    const int *len;
    char *ws;
    int *parent, *token, *node;
    double *score;
};

// the step's fp32 row value before normalisation: the input (modes 0, 1) or f[n, t] + g_slot (mode 2)
__device__ __forceinline__ float RowZ(const StepParams &P, long row, long frow, int k) {
    const float z = load_y(P.rows, P.dtype, row + k);
    return P.mode == 2 ? load_y(P.enc, P.dtype, frow + k) + z : z;
}

}  // namespace

}  // namespace ccb
