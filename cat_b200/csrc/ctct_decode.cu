// CTC-T (CTC-Transducer) prefix beam search: one launch per frame, one CTA per utterance (DESIGN.md §7 "CTC-T beam
// search").  Every frame emits one symbol, as in the CTC-T loss; a beam entry is a prefix with two fp64 masses, b (the last
// emission was blank, or nothing was emitted) and n (the last emission was the prefix's last token).  The caller runs the
// predictor and joiner networks between launches; each step reads the (N*B, V) row block of the current beam slots and
//   1. ranks each live row's non-blank entries: the k = min(B, V - 1) largest lp, ties to the lower token, exactly (one warp
//      per row, a windowed scan against the k-th best so far, bitonic-sorted in the warp's buffer when it fills);
//   2. forms the candidates of row r: extension (r, j) adds (c == last ? b : s) + lp[c] to n(prefix + c); the stay adds
//      s + lp[blank] to b(prefix) and n + lp[last] to n(prefix).  An extension whose prefix is a beam slot's folds into that
//      slot's stay (at most one does, the beam's prefixes being distinct); logaddexp in fp64, no atomics;
//   3. keeps the B best targets by (s = b (+) n desc, first-appearance key asc), key r(k+1)+j for an extension and r(k+1)+k
//      for a stay, a target's key the smaller of its contributions', by the same windowed scan over the key space;
//   4. writes the next beam in that rank order: parent slot, token (-1: the stay, or an extension folded into one), trie node
//      (created in rank order if missing), s; b and n stay in the workspace.
// The beam is ranked, so ccb_rnnt_beam_finish (rnnt_decode.cu) is the finish: its stable rank is the identity and it walks
// back the same trie.
#include "transducer_beam.cuh"

namespace ccb {

namespace {

constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
constexpr int kSort = 2048;                  // global selection: the best B, then the targets waiting to be sorted
constexpr int kWindow = 2 * kThreads;        // keys scanned between two looks at the buffer
constexpr int kRowBuf = 256;                 // per-warp row top-k: the best k (<= kBeamMax), then the waiting entries
constexpr int kNoKey = 0x7fffffff;
constexpr size_t kPoolBytes = (size_t)kWarps * kRowBuf * (sizeof(float) + sizeof(int));
static_assert(kPoolBytes >= (size_t)kSort * (sizeof(double) + sizeof(int)), "the row buffers and the sort share the pool");

// per utterance, after the N tries: b and n of every slot, then per (row r, rank j < k) the token, the extension's mass and
// the slot it folds into (-1: none)
__host__ __device__ __forceinline__ size_t CtctUttBytes(int B) { return Up256((size_t)B * (16 + 16 * (size_t)B)); }

struct CtctState {
    double *b, *n, *ext;
    int *tok, *fold;
};

__device__ __forceinline__ CtctState UttState(char *ws, int n, int N, int T, int B) {
    CtctState st;
    st.b = reinterpret_cast<double *>(ws + (size_t)N * UttBytes(T, B) + (size_t)n * CtctUttBytes(B));
    st.n = st.b + B;
    st.ext = st.n + B;
    st.tok = reinterpret_cast<int *>(st.ext + (size_t)B * B);
    st.fold = st.tok + (size_t)B * B;
    return st;
}

// the trie node (parent, tok), or -1
__device__ __forceinline__ int TrieFind(const Trie &tr, int parent, int tok) {
    for (unsigned h = TrieHash(parent, tok, tr.hslots);; h = (h + 1) & (unsigned)(tr.hslots - 1)) {
        const int x = tr.hash[h];
        if (x < 0) return -1;
        if (tr.parent[x] == parent && tr.tok[x] == tok) return x;
    }
}

// a ranks before b in a row: larger lp, then lower token
__device__ __forceinline__ bool RowBefore(float va, int ca, float vb, int cb) { return va > vb || (va == vb && ca < cb); }

// bitonic sort of v/c[0, P) into RowBefore order (P a power of two), by one warp
__device__ void WarpBitonicSort(float *v, int *c, int P, int lane) {
    for (int size = 2; size <= P; size <<= 1)
        for (int j = size >> 1; j > 0; j >>= 1) {
            for (int i = lane; i < P; i += 32) {
                const int x = i ^ j;
                if (x > i) {
                    const bool up = (i & size) == 0;
                    const bool sw = up ? RowBefore(v[x], c[x], v[i], c[i]) : RowBefore(v[i], c[i], v[x], c[x]);
                    if (sw) {
                        const float tv = v[i]; v[i] = v[x]; v[x] = tv;
                        const int tc = c[i]; c[i] = c[x]; c[x] = tc;
                    }
                }
            }
            __syncwarp();
        }
}

__global__ void __launch_bounds__(kThreads) ctct_beam_init_kernel(int N, int T, int B, char *ws) {
    const CtctState st = UttState(ws, blockIdx.x, N, T, B);
    for (int q = threadIdx.x; q < B; q += blockDim.x) {
        st.b[q] = kNegInf;
        st.n[q] = q == 0 ? 0.0 : kNegInf;
    }
}

__global__ void __launch_bounds__(kThreads) ctct_beam_step_kernel(const StepParams P) {
    __shared__ __align__(16) unsigned char s_pool[kPoolBytes];
    __shared__ double s_score[kBeamMax], s_b[kBeamMax], s_n[kBeamMax], s_stay[kBeamMax];
    __shared__ int s_node[kBeamMax], s_last[kBeamMax], s_key[kBeamMax], o_node[kBeamMax], o_tok[kBeamMax];
    __shared__ float s_lse[kBeamMax];
    __shared__ int s_nb, s_cnt, s_kept;
    double *sort_m = reinterpret_cast<double *>(s_pool);
    int *sort_k = reinterpret_cast<int *>(s_pool + kSort * sizeof(double));
    const int n = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int B = P.B, V = P.V, T = P.T, t = P.t;
    const int k = min(B, V - 1), K1 = k + 1;
    const size_t slot0 = (size_t)n * B;
    if (t >= P.len[n]) {   // the utterance has ended: every slot stays itself
        for (int q = tid; q < B; q += blockDim.x) { P.parent[slot0 + q] = q; P.token[slot0 + q] = -1; }
        return;
    }
    const Trie tr = UttTrie(P.ws, n, T, B);
    const CtctState st = UttState(P.ws, n, P.N, T, B);
    for (int q = tid; q < B; q += blockDim.x) {
        s_score[q] = P.score[slot0 + q];
        s_node[q] = P.node[slot0 + q];
        s_b[q] = st.b[q];
        s_n[q] = st.n[q];
        s_last[q] = s_node[q] >= 0 ? tr.tok[s_node[q]] : -1;
    }
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
    // row normalisers (modes 1, 2): the RNN-T step's, operation for operation, so that a row's lp is the same fp32 value in
    // both searches; one warp per row, an online (max, sum of exp) in fp32, merged in a fixed tree
    if (P.mode != 0) {
        for (int r = warp; r < nb; r += blockDim.x >> 5) {
            const long row = (long)(slot0 + r) * V;
            float m = -INFINITY, s = 0.f;
            for (int c = lane; c < V; c += 32) {
                const float z = RowZ(P, row, frow, c);
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
    // 1 + 2. per row (one warp each): the top-k tokens and their extension masses, the stay's b and n
    {
        float *bv = reinterpret_cast<float *>(s_pool) + warp * kRowBuf;
        int *bc = reinterpret_cast<int *>(s_pool + (size_t)kWarps * kRowBuf * sizeof(float)) + warp * kRowBuf;
        for (int r = warp; r < nb; r += kWarps) {
            const long row = (long)(slot0 + r) * V;
            const float z0 = P.mode != 0 ? s_lse[r] : 0.f;
            auto lp = [&](int c) {
                float v = RowZ(P, row, frow, c);
                if (P.mode != 0) v = v - z0;
                return v;
            };
            for (int i = lane; i < k; i += 32) { bv[i] = -INFINITY; bc[i] = kNoKey; }
            __syncwarp();
            float thr_v = -INFINITY;
            int thr_c = kNoKey, cnt = 0;
            for (int c0 = 0; k > 0 && c0 < V; c0 += 32) {
                const int c = c0 + lane;
                float v = 0.f;
                bool keep = false;
                if (c < V && c != P.blank) {
                    v = lp(c);
                    keep = RowBefore(v, c, thr_v, thr_c);
                }
                const unsigned mask = __ballot_sync(0xffffffffu, keep);
                if (keep) {
                    const int pos = k + cnt + __popc(mask & ((1u << lane) - 1u));
                    bv[pos] = v;
                    bc[pos] = c;
                }
                cnt += __popc(mask);
                if (cnt > kRowBuf - k - 32 || (cnt > 0 && c0 + 32 >= V)) {
                    const int ps = Pow2Ceil(k + cnt);
                    __syncwarp();
                    for (int i = k + cnt + lane; i < ps; i += 32) { bv[i] = -INFINITY; bc[i] = kNoKey; }
                    __syncwarp();
                    WarpBitonicSort(bv, bc, ps, lane);
                    cnt = 0;
                    thr_v = bv[k - 1];
                    thr_c = bc[k - 1];
                }
            }
            __syncwarp();
            const int last = s_last[r];
            const double s = s_score[r];
            for (int j = lane; j < k; j += 32) {
                const int c = bc[j];
                st.tok[(size_t)r * B + j] = c;
                st.ext[(size_t)r * B + j] = (c == last ? s_b[r] : s) + (double)bv[j];
                st.fold[(size_t)r * B + j] = -1;
            }
            __syncwarp();
            if (lane == 0) {
                s_b[r] = s + (double)lp(P.blank);   // the stay; s_b / s_n of row r are read only by this warp until here
                s_n[r] = last >= 0 ? s_n[r] + (double)lp(last) : kNegInf;
            }
            __syncwarp();
        }
    }
    __syncthreads();
    // the extension that produces slot q's prefix, if it is a candidate, folds into q's stay: q's key the smaller
    for (int q = tid; q < nb; q += blockDim.x) {
        int key = q * K1 + k;
        double nq = s_n[q];
        const int last = s_last[q];
        if (last >= 0 && k > 0) {
            const int pn = tr.parent[s_node[q]];
            for (int r = 0; r < nb; ++r) {
                if (s_node[r] != pn) continue;
                for (int j = 0; j < k; ++j)
                    if (st.tok[(size_t)r * B + j] == last) {
                        nq = lse(nq, st.ext[(size_t)r * B + j]);
                        key = min(key, r * K1 + j);
                        st.fold[(size_t)r * B + j] = q;
                        break;
                    }
                break;
            }
        }
        s_n[q] = nq;
        s_key[q] = key;
        s_stay[q] = lse(s_b[q], nq);
    }
    for (int i = tid; i < B; i += blockDim.x) { sort_m[i] = kNegInf; sort_k[i] = kNoKey; }   // the pool held the row buffers
    __syncthreads();
    // 3. exact top-B over the key space: each target at its own key, its mass s; the keys of folded extensions, and the stay
    // positions whose target took an extension's smaller key, hold no target
    const int total = nb * K1;
    const int cap = kSort - B;
    for (int w0 = 0; w0 < total; w0 += kWindow) {
        const double thr_m = sort_m[B - 1];
        const int thr_k = sort_k[B - 1];
        for (int f = w0 + tid; f < min(total, w0 + kWindow); f += blockDim.x) {
            const int r = f / K1, j = f - r * K1;
            const int q = j == k ? r : st.fold[(size_t)r * B + j];
            const double m = q < 0 ? st.ext[(size_t)r * B + j] : s_key[q] == f ? s_stay[q] : kNegInf;
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
        int kept = 0;
        while (kept < B && sort_m[kept] > kNegInf) ++kept;
        s_kept = kept;
    }
    __syncthreads();
    const int kept = s_kept;
    // 4. the next beam in rank order; the trie nodes of new extensions looked up, the missing ones created below
    for (int i = tid; i < kept; i += blockDim.x) {
        const int f = sort_k[i], r = f / K1, j = f - r * K1;
        const int q = j == k ? r : st.fold[(size_t)r * B + j];
        if (q >= 0) {   // a stay, possibly with a folded extension
            P.parent[slot0 + i] = q;
            o_tok[i] = -1;
            o_node[i] = s_node[q];
            st.b[i] = s_b[q];
            st.n[i] = s_n[q];
        } else {
            const int c = st.tok[(size_t)r * B + j];
            P.parent[slot0 + i] = r;
            o_tok[i] = c;
            o_node[i] = TrieFind(tr, s_node[r], c);
            st.b[i] = kNegInf;
            st.n[i] = sort_m[i];
        }
        P.token[slot0 + i] = o_tok[i];
        P.score[slot0 + i] = sort_m[i];
    }
    __syncthreads();
    if (tid == 0) {   // missing children created in rank order (distinct: the beam's prefixes are distinct)
        int next = *tr.next;
        for (int i = 0; i < kept; ++i) {
            if (o_node[i] >= 0) continue;
            const int par = s_node[P.parent[slot0 + i]], x = next++;
            tr.parent[x] = par; tr.tok[x] = o_tok[i];
            unsigned h = TrieHash(par, o_tok[i], tr.hslots);
            while (tr.hash[h] >= 0) h = (h + 1) & (unsigned)(tr.hslots - 1);
            tr.hash[h] = x;
            o_node[i] = x;
        }
        *tr.next = next;
    }
    __syncthreads();
    for (int q = tid; q < B; q += blockDim.x) {
        if (q < kept) {
            P.node[slot0 + q] = o_node[q];
        } else {
            P.parent[slot0 + q] = q; P.token[slot0 + q] = -1; P.node[slot0 + q] = -1; P.score[slot0 + q] = kNegInf;
            st.b[q] = kNegInf; st.n[q] = kNegInf;
        }
    }
}

}  // namespace

size_t CtctBeamWsBytes(int N, int T, int B) { return RnntBeamWsBytes(N, T, B) + (size_t)N * CtctUttBytes(B); }

int LaunchCtctBeamInit(int N, int T, int B, void *ws, int *parent, int *token, int *node, double *score, cudaStream_t s) {
    const int rc = LaunchRnntBeamInit(N, T, B, ws, parent, token, node, score, s);
    if (rc) return rc;
    ctct_beam_init_kernel<<<N, kThreads, 0, s>>>(N, T, B, reinterpret_cast<char *>(ws));
    CountLaunch();
    return (int)cudaGetLastError();
}

int LaunchCtctBeamStep(const void *rows, const void *enc, int dtype, int mode, int N, int T, int B, int V, int t,
                       const int *len, int blank, void *ws, int *parent, int *token, int *node, double *score, cudaStream_t s) {
    StepParams p;
    p.rows = rows; p.enc = enc; p.dtype = dtype; p.mode = mode;
    p.N = N; p.T = T; p.B = B; p.V = V; p.t = t; p.blank = blank;
    p.len = len; p.ws = reinterpret_cast<char *>(ws);
    p.parent = parent; p.token = token; p.node = node; p.score = score;
    ctct_beam_step_kernel<<<N, kThreads, 0, s>>>(p);
    CountLaunch();
    return (int)cudaGetLastError();
}

}  // namespace ccb
