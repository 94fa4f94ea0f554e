// RNN-T loss over the joint tensor in CAT's compact layout or the padded one, and the joiner's gather.sum (DESIGN.md §7
// "RNN-T loss").  Row pass -> alpha/beta pass (forward); gradient pass (backward).  No atomics anywhere: every output
// element has one writer and every sum a fixed order, so two identical calls give identical bits.
#include <algorithm>
#include <type_traits>

#include "common.cuh"

namespace ccb {
namespace {

constexpr int kRowThreads = 256;    // row and gradient passes: 8 warps per CTA
constexpr int kAbThreads = 256;     // alpha/beta pass: one CTA per (utterance, direction), threads over u
constexpr int kPrepThreads = 256;

size_t Align256(size_t b) { return (b + 255) / 256 * 256; }

// per utterance, in the workspace (rnnt_prep_kernel)
struct RnntMeta {
    long long roff;   // first row of the utterance's block
    long long loff;   // first label
    long long span;   // rows of the block, clamped to the tensor: what the gradient pass writes
    int T, U;         // lengths as given
    int ts;           // rows per frame: U + 1 (compact) or Umax + 1 (padded)
    int bad;          // lengths or labels invalid: NaN cost, zero gradient, rows never read
};

struct RnntLayout {
    size_t meta, tail, logp, alpha, beta, lpb, lpl, lpr, lse, total;
};

// ctct: the CTC-T loss's workspace, with two cells per row in each direction and the lpr block (lpr = 0 otherwise)
RnntLayout MakeRnntLayout(int N, long long rows, bool ctct) {
    const size_t states = ctct ? 2 : 1;
    RnntLayout L;
    size_t o = 0;
    L.meta = o;  o += Align256(sizeof(RnntMeta) * (size_t)N);
    L.tail = o;  o += 256;
    L.logp = o;  o += Align256(2 * sizeof(double) * (size_t)N);   // from alpha, then from beta
    L.alpha = o; o += Align256(states * sizeof(double) * (size_t)rows);
    L.beta = o;  o += Align256(states * sizeof(double) * (size_t)rows);
    L.lpb = o;   o += Align256(sizeof(float) * (size_t)rows);
    L.lpl = o;   o += Align256(sizeof(float) * (size_t)rows);
    L.lpr = 0;
    if (ctct) { L.lpr = o; o += Align256(sizeof(float) * (size_t)rows); }
    L.lse = o;   o += Align256(sizeof(float) * (size_t)rows);
    L.total = o;
    return L;
}

template <typename T> T *At(void *ws, size_t off) { return reinterpret_cast<T *>(reinterpret_cast<char *>(ws) + off); }
// a block that only the CTC-T layouts hold (lpr, PR: offset 0 otherwise), or nullptr
template <typename T> T *AtOpt(void *ws, size_t off) { return off ? At<T>(ws, off) : nullptr; }

// ------------------------------------------------------------------------------------------------
// 16-byte row chunks in a compile-time dtype (VEC) or single elements through load_y (rows whose byte length or base is not
// a multiple of 16)
// ------------------------------------------------------------------------------------------------
template <int DT> __host__ __device__ constexpr int EltBytes() { return DT == CCB_DTYPE_F32 ? 4 : 2; }
template <int DT, bool VEC> __host__ __device__ constexpr int ChunkElems() { return VEC ? 16 / EltBytes<DT>() : 1; }

template <int DT> __device__ __forceinline__ float From16(unsigned h) {
    return DT == CCB_DTYPE_BF16 ? __bfloat162float(__ushort_as_bfloat16((unsigned short)h))
                                : __half2float(__ushort_as_half((unsigned short)h));
}
template <int DT> __device__ __forceinline__ unsigned To16(float v) {
    return DT == CCB_DTYPE_BF16 ? __bfloat16_as_ushort(__float2bfloat16_rn(v)) : __half_as_ushort(__float2half_rn(v));
}

// chunk c of the row whose first element is `base`, read once (streaming)
template <int DT, bool VEC>
__device__ __forceinline__ void LoadChunk(const void *p, long long base, long long c, float *v) {
    if constexpr (!VEC) {
        v[0] = load_y(p, DT, base + c);
    } else if constexpr (DT == CCB_DTYPE_F32) {
        const float4 q = __ldcs(reinterpret_cast<const float4 *>(reinterpret_cast<const float *>(p) + base) + c);
        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    } else {
        const uint4 q = __ldcs(reinterpret_cast<const uint4 *>(reinterpret_cast<const unsigned short *>(p) + base) + c);
        const unsigned w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) { v[2 * i] = From16<DT>(w[i] & 0xffffu); v[2 * i + 1] = From16<DT>(w[i] >> 16); }
    }
}

template <int DT, bool VEC>
__device__ __forceinline__ void StoreChunk(void *p, long long base, long long c, const float *v) {
    if constexpr (!VEC) {
        store_y(p, DT, base + c, v[0]);
    } else if constexpr (DT == CCB_DTYPE_F32) {
        __stcs(reinterpret_cast<float4 *>(reinterpret_cast<float *>(p) + base) + c, make_float4(v[0], v[1], v[2], v[3]));
    } else {
        uint4 q;
        q.x = To16<DT>(v[0]) | (To16<DT>(v[1]) << 16); q.y = To16<DT>(v[2]) | (To16<DT>(v[3]) << 16);
        q.z = To16<DT>(v[4]) | (To16<DT>(v[5]) << 16); q.w = To16<DT>(v[6]) | (To16<DT>(v[7]) << 16);
        __stcs(reinterpret_cast<uint4 *>(reinterpret_cast<unsigned short *>(p) + base) + c, q);
    }
}

// (max, sum of exp(x - max)) pairs: the online logsumexp state; -inf max means "nothing finite seen"
__device__ __forceinline__ void LseMerge(float &m, float &s, float mo, float so) {
    const float mm = fmaxf(m, mo);
    if (mm == -INFINITY) return;
    s = s * __expf(m - mm) + so * __expf(mo - mm);
    m = mm;
}

__device__ __forceinline__ double LogAddD(double a, double b) {
    const double m = fmax(a, b);
    if (m == -INFINITY) return m;
    return m + log1p(exp(-fabs(a - b)));
}

// ------------------------------------------------------------------------------------------------
// Exclusive int64 prefix sums over the N utterances, one CTA, in chunks of kPrepThreads (fixed order: deterministic).  f(n) returns the two inputs of
// utterance n; g(n, ex0, ex1) receives their exclusive sums.  Returns the totals (on every thread).
// ------------------------------------------------------------------------------------------------
template <typename F, typename G>
__device__ void ScanUtts(int N, F f, G g, long long *tot0, long long *tot1) {
    constexpr int kWarps = kPrepThreads / 32;
    __shared__ longlong2 part[kWarps];
    __shared__ long long carry[2];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) { carry[0] = 0; carry[1] = 0; }
    __syncthreads();
    for (int base = 0; base < N; base += kPrepThreads) {
        const int n = base + (int)threadIdx.x;
        const longlong2 in = n < N ? f(n) : make_longlong2(0, 0);
        longlong2 inc = in;   // inclusive sums within the warp, then across warps
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long x = __shfl_up_sync(0xffffffffu, inc.x, o), y = __shfl_up_sync(0xffffffffu, inc.y, o);
            if (lane >= o) { inc.x += x; inc.y += y; }
        }
        if (lane == 31) part[warp] = inc;
        __syncthreads();
        long long wx = 0, wy = 0;
        for (int i = 0; i < warp; ++i) { wx += part[i].x; wy += part[i].y; }
        if (n < N) g(n, carry[0] + wx + inc.x - in.x, carry[1] + wy + inc.y - in.y);
        __syncthreads();
        if (threadIdx.x == kPrepThreads - 1) { carry[0] += wx + inc.x; carry[1] += wy + inc.y; }
        __syncthreads();
    }
    *tot0 = carry[0];
    *tot1 = carry[1];
}

// Per-utterance metadata from the device lengths.  Compact: rows (and labels) of utterance n follow those of n-1; padded:
// block n of Tmax (Umax+1) rows and row n of the (N, Umax) labels.  Negative lengths count as 0 in the offsets, so that
// the utterances' row ranges never overlap whatever the lengths are.
__global__ void __launch_bounds__(kPrepThreads) rnnt_prep_kernel(const int *lx, const int *ly, int N, long long rows,
                                                                 long long n_labels, int compact, int Tmax, int Umax,
                                                                 RnntMeta *meta, long long *tail) {
    auto in = [=](int n) {
        const long long T = max(lx[n], 0), U = max(ly[n], 0);
        return compact ? make_longlong2(T * (U + 1), U) : make_longlong2(0, 0);
    };
    auto out = [=](int n, long long roff, long long loff) {
        const int T = lx[n], U = ly[n];
        RnntMeta m;
        m.T = T; m.U = U;
        bool bad = T < 1 || U < 0;
        if (compact) {
            const long long own = (long long)max(T, 0) * (max(U, 0) + 1);
            m.roff = roff; m.loff = loff; m.ts = max(U, 0) + 1;
            m.span = min(own, max(rows - roff, 0LL));
            bad = bad || roff + own > rows;
        } else {
            m.ts = Umax + 1;
            m.span = (long long)Tmax * m.ts;
            m.roff = (long long)n * m.span; m.loff = (long long)n * Umax;
            bad = bad || T > Tmax || U > Umax;
        }
        bad = bad || m.loff + max(U, 0) > n_labels;
        m.bad = bad ? 1 : 0;
        meta[n] = m;
    };
    long long r_tot, l_tot;
    ScanUtts(N, in, out, &r_tot, &l_tot);
    if (threadIdx.x == 0) *tail = compact ? min(r_tot, rows) : rows;
}

// ------------------------------------------------------------------------------------------------
// Row pass.  Grid (row chunk, utterance): CTA (x, n) walks the rows t < T_n, u <= U_n of utterance n with stride gridDim.x.
// lpb = log p(blank), lpl = log p(y_{u+1}) (u < U_n); raw logits: minus the row's logsumexp, which is kept in lse.
// A label outside [0, V) or equal to blank marks the utterance bad (every writer writes 1; no atomics needed).
// CTCT (the CTC-T loss) also writes lpr = log p(y_u) (u >= 1), the repeat of the last label, read at the same row.
// ------------------------------------------------------------------------------------------------
// lp(row, y) - l for a label y of the utterance, or NaN (and the utterance marked bad) for an invalid one
__device__ __forceinline__ float LabelLp(const void *x, int dtype, long long V, long long row, int y, int blank, float l,
                                         RnntMeta *meta, int n) {
    if (y < 0 || y >= V || y == blank) { meta[n].bad = 1; return NAN; }
    return load_y(x, dtype, row * V + y) - l;
}

template <bool CTCT>
__device__ __forceinline__ void LpRows(const void *x, int dtype, long long V, const int *labels, int blank, RnntMeta *meta,
                                       float *lpb, float *lpl, float *lpr) {
    const int n = blockIdx.y;
    const RnntMeta m = meta[n];
    if (m.bad) return;
    const long long live = (long long)m.T * m.ts;
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < live; r += (long long)gridDim.x * blockDim.x) {
        const long long t = r / m.ts;
        const int u = (int)(r - t * m.ts);
        if (u > m.U) continue;
        const long long row = m.roff + r;
        lpb[row] = load_y(x, dtype, row * V + blank);
        if (u < m.U) {
            const int y = labels[m.loff + u];
            if (y < 0 || y >= V || y == blank) { meta[n].bad = 1; lpl[row] = NAN; }
            else lpl[row] = load_y(x, dtype, row * V + y);
        }
        if constexpr (CTCT) {
            if (u > 0) lpr[row] = LabelLp(x, dtype, V, row, labels[m.loff + u - 1], blank, 0.f, meta, n);
        }
    }
}

// One kernel for both losses, here and for the other bodies shared under CTCT (LogitRows, SimpleNorm, SimpleFixup,
// SimpleGrad): CTCT is the first template argument, so that a profile tells <false, ...> (RNN-T) from <true, ...> (CTC-T),
// and the RNN-T loss passes nullptr for lpr and PR.
template <bool CTCT>
__global__ void __launch_bounds__(kRowThreads) lp_rows_kernel(const void *x, int dtype, long long V, const int *labels,
                                                              int blank, RnntMeta *meta, float *lpb, float *lpl, float *lpr) {
    LpRows<CTCT>(x, dtype, V, labels, blank, meta, lpb, lpl, lpr);
}

template <int DT, bool VEC, bool CTCT>
__device__ __forceinline__ void LogitRows(const void *x, long long V, const int *labels, int blank, RnntMeta *meta, float *lpb,
                                          float *lpl, float *lpr, float *lse) {
    constexpr int K = ChunkElems<DT, VEC>();
    const int n = blockIdx.y;
    const RnntMeta m = meta[n];
    if (m.bad) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, W = blockDim.x >> 5;
    const long long live = (long long)m.T * m.ts, chunks = V / K;
    for (long long r = (long long)blockIdx.x * W + warp; r < live; r += (long long)gridDim.x * W) {
        const long long t = r / m.ts;
        const int u = (int)(r - t * m.ts);
        if (u > m.U) continue;
        const long long row = m.roff + r, base = row * V;
        float mx = -INFINITY, s = 0.f;
        for (long long c = lane; c < chunks; c += 32) {
            float v[K];
            LoadChunk<DT, VEC>(x, base, c, v);
            float cm = v[0];
#pragma unroll
            for (int i = 1; i < K; ++i) cm = fmaxf(cm, v[i]);
            if (cm == -INFINITY) continue;
            if (cm > mx) { s *= __expf(mx - cm); mx = cm; }
#pragma unroll
            for (int i = 0; i < K; ++i) s += __expf(v[i] - mx);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float mo = __shfl_xor_sync(0xffffffffu, mx, o), so = __shfl_xor_sync(0xffffffffu, s, o);
            LseMerge(mx, s, mo, so);
        }
        if (lane == 0) {
            const float l = mx == -INFINITY ? -INFINITY : mx + __logf(s);
            lse[row] = l;
            lpb[row] = load_y(x, DT, base + blank) - l;
            if (u < m.U) {
                const int y = labels[m.loff + u];
                if (y < 0 || y >= V || y == blank) { meta[n].bad = 1; lpl[row] = NAN; }
                else lpl[row] = load_y(x, DT, base + y) - l;
            }
            if constexpr (CTCT) {
                if (u > 0) lpr[row] = LabelLp(x, DT, V, row, labels[m.loff + u - 1], blank, l, meta, n);
            }
        }
    }
}

template <bool CTCT, int DT, bool VEC>
__global__ void __launch_bounds__(kRowThreads) logit_rows_kernel(const void *x, long long V, const int *labels, int blank,
                                                                 RnntMeta *meta, float *lpb, float *lpl, float *lpr, float *lse) {
    LogitRows<DT, VEC, CTCT>(x, V, labels, blank, meta, lpb, lpl, lpr, lse);
}

// ------------------------------------------------------------------------------------------------
// alpha / beta pass: CTA (n, 0) runs alpha, CTA (n, 1) beta, over anti-diagonals, threads over u; cells in fp64, kept per row
// in the workspace and read back by the next diagonal after the CTA barrier.
//   alpha(t,u) = logaddexp(alpha(t-1,u) + lpb(t-1,u), alpha(t,u-1) + lpl(t,u-1)),  log P = alpha(T-1,U) + lpb(T-1,U)
//   beta(t,u)  = logaddexp(beta(t+1,u) + lpb(t,u),   beta(t,u+1) + lpl(t,u)),     beta(T-1,U) = lpb(T-1,U), log P = beta(0,0)
// The parameters are ctct_alpha_beta_kernel's, so that one launch runs either; labels and lpr are not read.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kAbThreads) rnnt_alpha_beta_kernel(const RnntMeta *meta, const int *labels, const float *lpb,
                                                                     const float *lpl, const float *lpr, double *alpha,
                                                                     double *beta, double *logp, int N, float *costs,
                                                                     float *costs_beta) {
    const int n = blockIdx.x;
    const bool bwd = blockIdx.y == 1;
    const RnntMeta m = meta[n];
    if (m.bad) {
        if (threadIdx.x == 0) {
            logp[bwd ? N + n : n] = NAN;
            if (bwd) { if (costs_beta) costs_beta[n] = NAN; }
            else costs[n] = NAN;
        }
        return;
    }
    const int T = m.T, U = m.U;
    const long long ts = m.ts, off = m.roff;
    double *cell = bwd ? beta : alpha;
    for (int d = 0; d < T + U; ++d) {
        const int k_lo = max(0, d - (T - 1)), k_hi = min(U, d);
        for (int k = k_lo + (int)threadIdx.x; k <= k_hi; k += blockDim.x) {
            if (!bwd) {
                const int u = k, t = d - k;
                const long long r = off + t * ts + u;
                double a = 0.0;
                if (d > 0) {
                    const double x1 = t > 0 ? cell[r - ts] + (double)lpb[r - ts] : -INFINITY;
                    const double x2 = u > 0 ? cell[r - 1] + (double)lpl[r - 1] : -INFINITY;
                    a = LogAddD(x1, x2);
                }
                cell[r] = a;
            } else {
                const int u = U - k, t = (T - 1) - (d - k);
                const long long r = off + t * ts + u;
                double b = (double)lpb[r];
                if (d > 0) {
                    const double x1 = t < T - 1 ? cell[r + ts] + (double)lpb[r] : -INFINITY;
                    const double x2 = u < U ? cell[r + 1] + (double)lpl[r] : -INFINITY;
                    b = LogAddD(x1, x2);
                }
                cell[r] = b;
            }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        if (!bwd) {
            const long long last = off + (T - 1) * ts + U;
            const double lp = cell[last] + (double)lpb[last];
            logp[n] = lp;
            costs[n] = (float)-lp;
        } else {
            logp[N + n] = cell[off];
            if (costs_beta) costs_beta[n] = (float)-cell[off];
        }
    }
}

// The weighted posteriors of the blank and label transitions out of live cell (t, u) at workspace row `row` (formulas below);
// shared by the gradient pass and the LogAdd joiner's cell weights.
__device__ __forceinline__ void CellPosteriors(const RnntMeta &m, long long row, long long t, int u, const double *alpha,
                                               const double *beta, const float *lpb, const float *lpl, double lP, float wn,
                                               float &pb, float &pl) {
    const double a = alpha[row];
    pb = 0.f; pl = 0.f;
    if (t < m.T - 1) pb = (float)exp(a + (double)lpb[row] + beta[row + m.ts] - lP);
    else if (u == m.U) pb = (float)exp(a + (double)lpb[row] - lP);
    if (u < m.U) pl = (float)exp(a + (double)lpl[row] + beta[row + 1] - lP);
    pb *= wn; pl *= wn;
}

// ------------------------------------------------------------------------------------------------
// CTC-T alpha / beta pass (DESIGN.md §7 "CTC-T loss"): CTA (n, 0) runs alpha, CTA (n, 1) beta, frame by frame, threads over
// u, each thread both states of its u; one CTA barrier per frame.  Two fp64 cells per row and direction: state b (u labels,
// the last emission blank or nothing) at cell[2 row], state l (the last emission y_u) at cell[2 row + 1].  Row (t, u) keeps
// alpha_t(u, .), the states before frame t, and beta_{t+1}(u, .), the states after it:
//   alpha_{t+1}(u,b) = [alpha_t(u,b) + alpha_t(u,l)] lpb(t,u)
//   alpha_{t+1}(u,l) = alpha_t(u,l) lpr(t,u) + [alpha_t(u-1,b) + alpha_t(u-1,l) if u = 1 or y_u != y_{u-1}] lpl(t,u-1)
//   beta_t(u,b) = beta_{t+1}(u,b) lpb(t,u) + beta_{t+1}(u+1,l) lpl(t,u)
//   beta_t(u,l) = beta_{t+1}(u,b) lpb(t,u) + beta_{t+1}(u,l) lpr(t,u) + [beta_{t+1}(u+1,l) lpl(t,u) if y_{u+1} != y_u]
// (+ is logaddexp, juxtaposition a product of probabilities), alpha_0(0,b) = 0, beta_T(U,.) = 0, every other boundary cell
// -inf, and log P = alpha_T(U,b) + alpha_T(U,l) = beta_0(0,b).  An infeasible utterance gets log P = -inf, cost +inf.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kAbThreads) ctct_alpha_beta_kernel(const RnntMeta *meta, const int *labels, const float *lpb,
                                                                     const float *lpl, const float *lpr, double *alpha,
                                                                     double *beta, double *logp, int N, float *costs,
                                                                     float *costs_beta) {
    const int n = blockIdx.x;
    const bool bwd = blockIdx.y == 1;
    const RnntMeta m = meta[n];
    if (m.bad) {
        if (threadIdx.x == 0) {
            logp[bwd ? N + n : n] = NAN;
            if (bwd) { if (costs_beta) costs_beta[n] = NAN; }
            else costs[n] = NAN;
        }
        return;
    }
    const int T = m.T, U = m.U;
    const long long ts = m.ts, off = m.roff;
    const int *y = labels + m.loff;     // y[u - 1] = y_u
    double *cell = bwd ? beta : alpha;
    double eb = -INFINITY, el = -INFINITY;   // the end state the thread owning u = U (alpha) or u = 0 (beta) returns
    if (!bwd) {
        for (int u = threadIdx.x; u <= U; u += blockDim.x) {
            cell[2 * (off + u)] = u == 0 ? 0.0 : -INFINITY;
            cell[2 * (off + u) + 1] = -INFINITY;
        }
        __syncthreads();
        for (int t = 0; t < T; ++t) {
            for (int u = threadIdx.x; u <= U; u += blockDim.x) {
                const long long r = off + t * ts + u;
                const double ab = cell[2 * r], al = cell[2 * r + 1];
                const double nb = LogAddD(ab, al) + (double)lpb[r];
                double nl = -INFINITY;
                if (u > 0) {
                    const double pb = cell[2 * (r - 1)], pl = cell[2 * (r - 1) + 1];
                    const double src = u == 1 || y[u - 1] != y[u - 2] ? LogAddD(pb, pl) : pb;
                    nl = LogAddD(al + (double)lpr[r], src + (double)lpl[r - 1]);
                }
                if (t + 1 < T) { cell[2 * (r + ts)] = nb; cell[2 * (r + ts) + 1] = nl; }
                else if (u == U) { eb = nb; el = nl; }
            }
            __syncthreads();
        }
        if (threadIdx.x == U % blockDim.x) {
            const double lp = LogAddD(eb, el);
            logp[n] = lp;
            costs[n] = (float)-lp;
        }
    } else {
        for (int u = threadIdx.x; u <= U; u += blockDim.x) {
            const long long r = off + (T - 1) * ts + u;
            cell[2 * r] = u == U ? 0.0 : -INFINITY;
            cell[2 * r + 1] = u == U && U > 0 ? 0.0 : -INFINITY;
        }
        __syncthreads();
        for (int t = T - 1; t >= 0; --t) {
            for (int u = threadIdx.x; u <= U; u += blockDim.x) {
                const long long r = off + t * ts + u;
                const double xb = cell[2 * r] + (double)lpb[r];
                const double xn = u < U ? cell[2 * (r + 1) + 1] + (double)lpl[r] : -INFINITY;
                const double nb = LogAddD(xb, xn);
                double nl = -INFINITY;
                if (u > 0) {
                    nl = LogAddD(xb, cell[2 * r + 1] + (double)lpr[r]);
                    if (u < U && y[u] != y[u - 1]) nl = LogAddD(nl, xn);
                }
                if (t > 0) { cell[2 * (r - ts)] = nb; cell[2 * (r - ts) + 1] = nl; }
                else if (u == 0) eb = nb;
            }
            __syncthreads();
        }
        if (threadIdx.x == 0) {
            logp[N + n] = eb;
            if (costs_beta) costs_beta[n] = (float)-eb;
        }
    }
}

// The weighted posteriors of the three CTC-T transitions that read live row (t, u) at workspace row `row`: pb (blank, into
// (u,b)), pr (the repeat of y_u, into (u,l), u >= 1) and pl (y_{u+1}, into (u+1,l), u < U; from (u,l) too unless
// y_{u+1} = y_u).  All zero when log P = -inf (no path).  Shared by the gradient pass and the LogAdd joiner's cell weights.
__device__ __forceinline__ void CtctPosteriors(const RnntMeta &m, const int *labels, long long row, int u, const double *alpha,
                                               const double *beta, const float *lpb, const float *lpl, const float *lpr,
                                               double lP, float wn, float &pb, float &pr, float &pl) {
    pb = 0.f; pr = 0.f; pl = 0.f;
    if (lP == -INFINITY) return;
    const double ab = alpha[2 * row], al = alpha[2 * row + 1];   // the two source states, summed as probabilities
    const double cb = (double)lpb[row] + beta[2 * row] - lP;
    pb = (float)(exp(ab + cb) + exp(al + cb));
    if (u > 0) pr = (float)exp(al + (double)lpr[row] + beta[2 * row + 1] - lP);
    if (u < m.U) {
        const bool rep = u > 0 && labels[m.loff + u] == labels[m.loff + u - 1];
        const double cl = (double)lpl[row] + beta[2 * (row + 1) + 1] - lP;
        pl = (float)(exp(ab + cl) + (rep ? 0.0 : exp(al + cl)));
    }
    pb *= wn; pr *= wn; pl *= wn;
}

// ------------------------------------------------------------------------------------------------
// Gradient pass: one warp per row, every row of the tensor written once.  Grid (row chunk, N + 1): CTA (x, n < N) walks
// utterance n's span (rows outside t < T_n, u <= U_n, and every row of a bad utterance, get zeros and are not read);
// CTA (x, N) zeroes the compact tail behind the last utterance.  With w = w_n,
//   pb = w exp(alpha + lpb + beta(t+1,u) - log P)   (at t = T-1 only for u = U, as exp(alpha + lpb - log P))
//   pl = w exp(alpha + lpl + beta(t,u+1) - log P)   (u < U)
//   grad[k] = [raw: exp(z_k - lse) (pb + pl)] - pb [k == blank] - pl [k == y_{u+1}]
// The parameters are ctct_grad_kernel's; lpr is not read.
// ------------------------------------------------------------------------------------------------
template <int DT, bool VEC, bool RAW>
__global__ void __launch_bounds__(kRowThreads) rnnt_grad_kernel(const void *x, long long V, const int *labels, int blank, int N,
                                                                const RnntMeta *meta, const long long *tail, long long rows,
                                                                const double *alpha, const double *beta, const double *logp,
                                                                const float *lpb, const float *lpl, const float *lpr,
                                                                const float *lse, const float *w, void *grad) {
    constexpr int K = ChunkElems<DT, VEC>();
    const int n = blockIdx.y;
    const bool utt = n < N;
    RnntMeta m{};
    long long first, count;
    if (utt) { m = meta[n]; first = m.roff; count = m.span; }
    else { first = *tail; count = rows - first; }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, W = blockDim.x >> 5;
    const long long chunks = V / K;
    const float wn = utt && !m.bad ? w[n] : 0.f;
    const double lP = utt && !m.bad ? logp[n] : 0.0;
    for (long long r = (long long)blockIdx.x * W + warp; r < count; r += (long long)gridDim.x * W) {
        const long long row = first + r, base = row * V;
        float pb = 0.f, pl = 0.f, l = 0.f;
        int y = -1;
        bool live = false;
        if (utt && !m.bad) {
            const long long t = r / m.ts;
            const int u = (int)(r - t * m.ts);
            if (t < m.T && u <= m.U) {
                live = true;
                CellPosteriors(m, row, t, u, alpha, beta, lpb, lpl, lP, wn, pb, pl);
                if (u < m.U) y = labels[m.loff + u];
                if constexpr (RAW) l = lse[row];
            }
        }
        const float occ = pb + pl;
        for (long long c = lane; c < chunks; c += 32) {
            float v[K];
            if (RAW && live) {
                LoadChunk<DT, VEC>(x, base, c, v);
#pragma unroll
                for (int i = 0; i < K; ++i) v[i] = __expf(v[i] - l) * occ;
            } else {
#pragma unroll
                for (int i = 0; i < K; ++i) v[i] = 0.f;
            }
            if (live) {
#pragma unroll
                for (int i = 0; i < K; ++i) {
                    const long long k = c * K + i;
                    if (k == blank) v[i] -= pb;
                    if (k == y) v[i] -= pl;
                }
            }
            StoreChunk<DT, VEC>(grad, base, c, v);
        }
    }
}

// CTC-T gradient pass: the RNN-T gradient pass with pb, pr and pl from CtctPosteriors,
//   grad[k] = [raw: exp(z_k - lse) (pb + pr + pl)] - pb [k == blank] - pr [k == y_u] - pl [k == y_{u+1}],
// where y_u = y_{u+1} puts both label terms on one element, in that order.
template <int DT, bool VEC, bool RAW>
__global__ void __launch_bounds__(kRowThreads) ctct_grad_kernel(const void *x, long long V, const int *labels, int blank, int N,
                                                                const RnntMeta *meta, const long long *tail, long long rows,
                                                                const double *alpha, const double *beta, const double *logp,
                                                                const float *lpb, const float *lpl, const float *lpr,
                                                                const float *lse, const float *w, void *grad) {
    constexpr int K = ChunkElems<DT, VEC>();
    const int n = blockIdx.y;
    const bool utt = n < N;
    RnntMeta m{};
    long long first, count;
    if (utt) { m = meta[n]; first = m.roff; count = m.span; }
    else { first = *tail; count = rows - first; }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, W = blockDim.x >> 5;
    const long long chunks = V / K;
    const float wn = utt && !m.bad ? w[n] : 0.f;
    const double lP = utt && !m.bad ? logp[n] : 0.0;
    // (t, u) of row r stepped along with r in 32-bit arithmetic: a 64-bit division here is a subroutine call, and the call
    // costs this kernel its registers (spills)
    const unsigned ts = utt ? (unsigned)m.ts : 1u, r0 = blockIdx.x * W + warp, step = gridDim.x * W;
    const unsigned dt = step / ts, du = step % ts;
    long long t = r0 / ts;
    unsigned uq = r0 % ts;
    for (long long r = r0; r < count; r += step, t += dt, uq += du) {
        if (uq >= ts) { uq -= ts; ++t; }
        const long long row = first + r, base = row * V;
        float pb = 0.f, pr = 0.f, pl = 0.f, l = 0.f;
        int y = -1, yr = -1;
        bool live = false;
        if (utt && !m.bad) {
            const int u = (int)uq;
            if (t < m.T && u <= m.U) {
                live = true;
                CtctPosteriors(m, labels, row, u, alpha, beta, lpb, lpl, lpr, lP, wn, pb, pr, pl);
                if (u > 0) yr = labels[m.loff + u - 1];
                if (u < m.U) y = labels[m.loff + u];
                if constexpr (RAW) l = lse[row];
            }
        }
        const float occ = pb + pr + pl;
        for (long long c = lane; c < chunks; c += 32) {
            float v[K];
            if (RAW && live) {
                LoadChunk<DT, VEC>(x, base, c, v);
#pragma unroll
                for (int i = 0; i < K; ++i) v[i] = __expf(v[i] - l) * occ;
            } else {
#pragma unroll
                for (int i = 0; i < K; ++i) v[i] = 0.f;
            }
            if (live) {
#pragma unroll
                for (int i = 0; i < K; ++i) {
                    const long long k = c * K + i;
                    if (k == blank) v[i] -= pb;
                    if (k == yr) v[i] -= pr;
                    if (k == y) v[i] -= pl;
                }
            }
            StoreChunk<DT, VEC>(grad, base, c, v);
        }
    }
}

// the gradient pass of either loss, whose kernels share ctct_grad_kernel's parameters
template <bool CTCT, int DT, bool VEC, bool RAW> auto GradKernel() {
    return CTCT ? ctct_grad_kernel<DT, VEC, RAW> : rnnt_grad_kernel<DT, VEC, RAW>;
}

// ------------------------------------------------------------------------------------------------
// gather.sum: out[off_n + t lb_n + u][h] = a[ta_n + t][h] + b[ub_n + u][h]; one warp per output row.  Backward: grad_a by a
// sum over u (contiguous rows), grad_b by a sum over t (rows at stride lb_n), each a fixed-order fp32 sum per (row, h).
// ------------------------------------------------------------------------------------------------
struct GatherMeta {
    long long off, ta, ub;
    int la, lb;
};

__global__ void __launch_bounds__(kPrepThreads) gather_prep_kernel(const int *la, const int *lb, int N, GatherMeta *meta) {
    // the scan carries (a rows, b rows); the output offset is a second pass of the same scan
    auto in = [=](int n) { return make_longlong2(max(la[n], 0), max(lb[n], 0)); };
    auto out = [=](int n, long long ta, long long ub) {
        meta[n].ta = ta; meta[n].ub = ub; meta[n].la = max(la[n], 0); meta[n].lb = max(lb[n], 0);
    };
    long long t0, t1;
    ScanUtts(N, in, out, &t0, &t1);
    auto in2 = [=](int n) { return make_longlong2((long long)max(la[n], 0) * max(lb[n], 0), 0); };
    auto out2 = [=](int n, long long off, long long) { meta[n].off = off; };
    __syncthreads();
    ScanUtts(N, in2, out2, &t0, &t1);
}

template <int DT>
__global__ void __launch_bounds__(kRowThreads) gather_sum_kernel(const void *a, const void *b, int H, const GatherMeta *meta,
                                                                 void *out) {
    const GatherMeta m = meta[blockIdx.y];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, W = blockDim.x >> 5;
    const long long count = (long long)m.la * m.lb;
    for (long long r = (long long)blockIdx.x * W + warp; r < count; r += (long long)gridDim.x * W) {
        const long long t = r / m.lb, u = r - t * m.lb;
        const long long ra = (m.ta + t) * H, rb = (m.ub + u) * H, ro = (m.off + r) * H;
        for (int h = lane; h < H; h += 32) store_y(out, DT, ro + h, load_y(a, DT, ra + h) + load_y(b, DT, rb + h));
    }
}

// grad_a (by_t = true: rows ta_n + t, summing over u) or grad_b (rows ub_n + u, summing over t); threads over h
template <int DT>
__global__ void __launch_bounds__(kRowThreads) gather_sum_bwd_kernel(const void *g, int H, const GatherMeta *meta, bool by_t,
                                                                     void *grad) {
    const GatherMeta m = meta[blockIdx.y];
    const int outer = by_t ? m.la : m.lb, inner = by_t ? m.lb : m.la;
    const long long step = by_t ? 1 : m.lb;
    for (int i = blockIdx.x; i < outer; i += gridDim.x) {
        const long long r0 = m.off + (by_t ? (long long)i * m.lb : i), dst = (by_t ? m.ta : m.ub) + i;
        for (int h = threadIdx.x; h < H; h += blockDim.x) {
            float acc = 0.f;
            for (int j = 0; j < inner; ++j) acc += load_y(g, DT, (r0 + j * step) * H + h);
            store_y(grad, DT, dst * H + h, acc);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// RNN-T loss of CAT's LogAdd joiner (DESIGN.md §7 "RNN-T loss, LogAdd joiner") from f (N, Tmax, V) and g (N, Umax+1, V),
// without the joint: z(t,u,k) = f[t,k] + g[u,k], Z(t,u) = logsumexp_k z = mf_t + mg_u + log S(t,u) with the row maxima mf, mg
// and S = sum_k Ef[t,k] Eg[u,k], Ef = exp(f - mf), Eg = exp(g - mg): one fp32 GEMM per utterance.  The lattice cells are the
// padded layout's (rnnt_prep_kernel with compact = 0, rnnt_alpha_beta_kernel as they are).  A cell with S < 2^-64 (the
// peaks of f[t] and g[u] on different tokens) is flagged and gets its Z from an exact logsumexp over f[t] + g[u] instead:
// the terms the GEMM flushes to zero are each below 2^-126, so for S >= 2^-64 they are below 2^-46 S for V <= 2^16.
// ------------------------------------------------------------------------------------------------
constexpr float kSimpleTiny = 0x1p-64f;
__device__ __forceinline__ bool SimpleFlagged(float s) { return !(s >= kSimpleTiny); }
// a row maximum as the exponent's offset: a row of -inf exponentiates to zeros, not NaN
__device__ __forceinline__ float SimpleOffset(float m) { return m == -INFINITY ? 0.f : m; }

struct SimpleLayout {
    RnntLayout r;                                     // meta .. lse over the N Tmax (Umax+1) cells; lse holds Z
    size_t mf, mg, ff, fg, S, W, PB, PL, PR, total;   // row maxima and "row has a flagged cell" of f and g; per cell S, W,
};                                                    // pb, pl (and pr for the CTC-T loss; PR = 0 otherwise)

SimpleLayout MakeSimpleLayout(int N, int Tmax, int Umax, bool ctct) {
    const size_t nf = (size_t)N * Tmax, ng = (size_t)N * (Umax + 1), cells = nf * (Umax + 1);
    SimpleLayout L;
    L.r = MakeRnntLayout(N, (long long)cells, ctct);
    size_t o = L.r.total;
    L.mf = o; o += Align256(sizeof(float) * nf);
    L.mg = o; o += Align256(sizeof(float) * ng);
    L.ff = o; o += Align256(sizeof(int) * nf);
    L.fg = o; o += Align256(sizeof(int) * ng);
    L.S = o;  o += Align256(sizeof(float) * cells);
    L.W = o;  o += Align256(sizeof(float) * cells);
    L.PB = o; o += Align256(sizeof(float) * cells);
    L.PL = o; o += Align256(sizeof(float) * cells);
    L.PR = 0;
    if (ctct) { L.PR = o; o += Align256(sizeof(float) * cells); }
    L.total = o;
    return L;
}

// Row maxima: one warp per live row, of f (blockIdx.z = 0, t < T_n) or of g (z = 1, u <= U_n); also clears the row's flag.
template <int DT, bool VEC>
__global__ void __launch_bounds__(kRowThreads) simple_rowmax_kernel(const void *f, const void *g, long long V, int Tmax, int Umax,
                                                                    const RnntMeta *meta, float *mf, float *mg, int *ff, int *fg) {
    constexpr int K = ChunkElems<DT, VEC>();
    const int n = blockIdx.y;
    const RnntMeta m = meta[n];
    if (m.bad) return;
    const bool is_g = blockIdx.z == 1;
    const int live = is_g ? m.U + 1 : m.T;
    const long long first = is_g ? (long long)n * (Umax + 1) : (long long)n * Tmax, chunks = V / K;
    const void *x = is_g ? g : f;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, W = blockDim.x >> 5;
    for (int r = blockIdx.x * W + warp; r < live; r += gridDim.x * W) {
        const long long base = (first + r) * V;
        float mx = -INFINITY;
        for (long long c = lane; c < chunks; c += 32) {
            float v[K];
            LoadChunk<DT, VEC>(x, base, c, v);
#pragma unroll
            for (int i = 0; i < K; ++i) mx = fmaxf(mx, v[i]);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if (lane == 0) {
            (is_g ? mg : mf)[first + r] = mx;
            (is_g ? fg : ff)[first + r] = 0;
        }
    }
}

// Normaliser GEMM: CTA (t tile, u tile, n) sums S(t,u) = sum_k Ef[t,k] Eg[u,k] over kSK-wide slabs of k, in increasing k, each
// thread a 4 x 2 block of cells in fp32 FFMA.  Tiles wholly past T_n or U_n + 1 return at once.  Epilogue per live cell: S;
// the label check (a label outside [0, V) or equal to blank marks the utterance bad, as the row pass does); then for an
// unflagged cell Z (in lse), lpb = z(blank) - Z and lpl = z(y_{u+1}) - Z, and for a flagged one the flags of rows t and u.
// CTCT also writes lpr = z(y_u) - Z (u >= 1) for an unflagged cell; an invalid y_u is skipped here (the cell of u - 1
// marks the utterance bad).
constexpr int kST = 64, kSU = 32, kSK = 32;
template <int DT, bool CTCT>
__device__ __forceinline__ void SimpleNorm(const void *f, const void *g, long long V, int Tmax, int Umax, const int *labels,
                                           int blank, RnntMeta *meta, const float *mf, const float *mg, int *ff, int *fg,
                                           float *S, float *lpb, float *lpl, float *lpr, float *lse) {
    const int n = blockIdx.z;
    const RnntMeta m = meta[n];
    const int t0 = blockIdx.x * kST, u0 = blockIdx.y * kSU;
    if (m.bad || t0 >= m.T || u0 > m.U) return;
    __shared__ float As[kSK][kST + 1], Bs[kSK][kSU + 1];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4, lk = tid & 31, lr = tid >> 5;
    const long long fr0 = (long long)n * Tmax, gr0 = (long long)n * (Umax + 1);
    float oa[kST / 8], ob[kSU / 8];      // the loader's rows lr + 8 i: their offsets (row maxima)
#pragma unroll
    for (int i = 0; i < kST / 8; ++i) { const int t = t0 + lr + 8 * i; oa[i] = t < m.T ? SimpleOffset(mf[fr0 + t]) : 0.f; }
#pragma unroll
    for (int i = 0; i < kSU / 8; ++i) { const int u = u0 + lr + 8 * i; ob[i] = u <= m.U ? SimpleOffset(mg[gr0 + u]) : 0.f; }
    float acc[4][2] = {};
    for (long long k0 = 0; k0 < V; k0 += kSK) {
        const long long k = k0 + lk;
#pragma unroll
        for (int i = 0; i < kST / 8; ++i) {
            const int r = lr + 8 * i, t = t0 + r;
            As[lk][r] = t < m.T && k < V ? expf(load_y(f, DT, (fr0 + t) * V + k) - oa[i]) : 0.f;
        }
#pragma unroll
        for (int i = 0; i < kSU / 8; ++i) {
            const int r = lr + 8 * i, u = u0 + r;
            Bs[lk][r] = u <= m.U && k < V ? expf(load_y(g, DT, (gr0 + u) * V + k) - ob[i]) : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int kk = 0; kk < kSK; ++kk) {
            float a[4], b[2];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = As[kk][ty + 16 * i];
#pragma unroll
            for (int j = 0; j < 2; ++j) b[j] = Bs[kk][tx + 16 * j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 2; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int t = t0 + ty + 16 * i;
        if (t >= m.T) continue;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int u = u0 + tx + 16 * j;
            if (u > m.U) continue;
            const long long row = m.roff + (long long)t * m.ts + u, fb = (fr0 + t) * V, gb = (gr0 + u) * V;
            const float s = acc[i][j];
            S[row] = s;
            int y = -1;
            if (u < m.U) {
                y = labels[m.loff + u];
                if (y < 0 || y >= V || y == blank) { meta[n].bad = 1; lpl[row] = NAN; continue; }
            }
            if (SimpleFlagged(s)) { ff[fr0 + t] = 1; fg[gr0 + u] = 1; continue; }
            const float Z = mf[fr0 + t] + mg[gr0 + u] + logf(s);
            lse[row] = Z;
            lpb[row] = (load_y(f, DT, fb + blank) + load_y(g, DT, gb + blank)) - Z;
            if (y >= 0) lpl[row] = (load_y(f, DT, fb + y) + load_y(g, DT, gb + y)) - Z;
            if constexpr (CTCT) {
                if (u > 0) {
                    const int yr = labels[m.loff + u - 1];
                    if (yr >= 0 && yr < V && yr != blank) lpr[row] = (load_y(f, DT, fb + yr) + load_y(g, DT, gb + yr)) - Z;
                }
            }
        }
    }
}

template <bool CTCT, int DT>
__global__ void __launch_bounds__(256) simple_norm_kernel(const void *f, const void *g, long long V, int Tmax, int Umax,
                                                          const int *labels, int blank, RnntMeta *meta, const float *mf,
                                                          const float *mg, int *ff, int *fg, float *S, float *lpb, float *lpl,
                                                          float *lpr, float *lse) {
    SimpleNorm<DT, CTCT>(f, g, V, Tmax, Umax, labels, blank, meta, mf, mg, ff, fg, S, lpb, lpl, lpr, lse);
}

// Underflow fix-up: one warp per flagged cell (rows t without a flagged cell are skipped by their flag) takes the exact
// logsumexp of f[t] + g[u] by an online max / sum, and rewrites Z, lpb and lpl (and lpr when CTCT).
template <int DT, bool VEC, bool CTCT>
__device__ __forceinline__ void SimpleFixup(const void *f, const void *g, long long V, int Tmax, int Umax, const int *labels,
                                            int blank, const RnntMeta *meta, const int *ff, const float *S, float *lpb,
                                            float *lpl, float *lpr, float *lse) {
    constexpr int K = ChunkElems<DT, VEC>();
    const int n = blockIdx.y;
    const RnntMeta m = meta[n];
    if (m.bad) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, W = blockDim.x >> 5;
    const long long live = (long long)m.T * m.ts, chunks = V / K, fr0 = (long long)n * Tmax, gr0 = (long long)n * (Umax + 1);
    for (long long r = (long long)blockIdx.x * W + warp; r < live; r += (long long)gridDim.x * W) {
        const long long t = r / m.ts;
        const int u = (int)(r - t * m.ts);
        const long long row = m.roff + r;
        if (u > m.U || !ff[fr0 + t] || !SimpleFlagged(S[row])) continue;
        const long long fb = (fr0 + t) * V, gb = (gr0 + u) * V;
        float mx = -INFINITY, s = 0.f;
        for (long long c = lane; c < chunks; c += 32) {
            float v[K], w[K];
            LoadChunk<DT, VEC>(f, fb, c, v);
            LoadChunk<DT, VEC>(g, gb, c, w);
            float cm = -INFINITY;
#pragma unroll
            for (int i = 0; i < K; ++i) { v[i] += w[i]; cm = fmaxf(cm, v[i]); }
            if (cm == -INFINITY) continue;
            if (cm > mx) { s *= expf(mx - cm); mx = cm; }
#pragma unroll
            for (int i = 0; i < K; ++i) s += expf(v[i] - mx);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float mo = __shfl_xor_sync(0xffffffffu, mx, o), so = __shfl_xor_sync(0xffffffffu, s, o);
            const float mm = fmaxf(mx, mo);
            if (mm != -INFINITY) { s = s * expf(mx - mm) + so * expf(mo - mm); mx = mm; }
        }
        if (lane == 0) {
            const float Z = mx == -INFINITY ? -INFINITY : mx + logf(s);
            lse[row] = Z;
            lpb[row] = (load_y(f, DT, fb + blank) + load_y(g, DT, gb + blank)) - Z;
            if (u < m.U) {
                const int y = labels[m.loff + u];
                lpl[row] = (load_y(f, DT, fb + y) + load_y(g, DT, gb + y)) - Z;
            }
            if constexpr (CTCT) {
                if (u > 0) {
                    const int y = labels[m.loff + u - 1];
                    lpr[row] = (load_y(f, DT, fb + y) + load_y(g, DT, gb + y)) - Z;
                }
            }
        }
    }
}

template <bool CTCT, int DT, bool VEC>
__global__ void __launch_bounds__(kRowThreads) simple_fixup_kernel(const void *f, const void *g, long long V, int Tmax, int Umax,
                                                                   const int *labels, int blank, const RnntMeta *meta,
                                                                   const int *ff, const float *S, float *lpb, float *lpl,
                                                                   float *lpr, float *lse) {
    SimpleFixup<DT, VEC, CTCT>(f, g, V, Tmax, Umax, labels, blank, meta, ff, S, lpb, lpl, lpr, lse);
}

// Cell weights: per live cell pb, pl (weighted posteriors, as the gradient pass) and W = (pb + pl) / S, 0 for a flagged cell.
// The parameters are ctct_simple_weights_kernel's; labels, lpr and PR are not used.
__global__ void __launch_bounds__(kRowThreads) simple_weights_kernel(const RnntMeta *meta, const int *labels, const double *alpha,
                                                                     const double *beta, const double *logp, const float *lpb,
                                                                     const float *lpl, const float *lpr, const float *S,
                                                                     const float *w, float *W, float *PB, float *PL,
                                                                     float *PR) {
    const int n = blockIdx.y;
    const RnntMeta m = meta[n];
    if (m.bad) return;
    const float wn = w[n];
    const double lP = logp[n];
    const long long live = (long long)m.T * m.ts;
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < live; r += (long long)gridDim.x * blockDim.x) {
        const long long t = r / m.ts;
        const int u = (int)(r - t * m.ts);
        if (u > m.U) continue;
        const long long row = m.roff + r;
        float pb, pl;
        CellPosteriors(m, row, t, u, alpha, beta, lpb, lpl, lP, wn, pb, pl);
        const float s = S[row];
        PB[row] = pb;
        PL[row] = pl;
        W[row] = SimpleFlagged(s) ? 0.f : (pb + pl) / s;
    }
}

// CTC-T cell weights: per live cell pb, pr, pl (CtctPosteriors) and W = (pb + pr + pl) / S, 0 for a flagged cell.
__global__ void __launch_bounds__(kRowThreads) ctct_simple_weights_kernel(const RnntMeta *meta, const int *labels,
                                                                          const double *alpha, const double *beta,
                                                                          const double *logp, const float *lpb,
                                                                          const float *lpl, const float *lpr, const float *S,
                                                                          const float *w, float *W, float *PB, float *PL,
                                                                          float *PR) {
    const int n = blockIdx.y;
    const RnntMeta m = meta[n];
    if (m.bad) return;
    const float wn = w[n];
    const double lP = logp[n];
    const long long live = (long long)m.T * m.ts;
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < live; r += (long long)gridDim.x * blockDim.x) {
        const long long t = r / m.ts;
        const int u = (int)(r - t * m.ts);
        if (u > m.U) continue;
        const long long row = m.roff + r;
        float pb, pr, pl;
        CtctPosteriors(m, labels, row, u, alpha, beta, lpb, lpl, lpr, lP, wn, pb, pr, pl);
        const float s = S[row];
        PB[row] = pb;
        PR[row] = pr;
        PL[row] = pl;
        W[row] = SimpleFlagged(s) ? 0.f : (pb + pr + pl) / s;
    }
}

// Gradient GEMM.  GF: grad_f, output rows r = t and reduction q = u; else grad_g, r = u and q = t.  With "own" the input
// whose gradient is written and "other" the one summed over,
//   grad[r,k] = E_own[r,k] sum_q W(r,q) E_other[q,k]  +  sum_{q flagged} (pb + pl) exp(z - Z)
//               - [k = blank] sum_q pb  -  sum_q pl [k = y_{u+1}],
// each sum over increasing q in fp32.  CTA (k tile, r tile, n) writes its whole kGR x kGC block: rows past the utterance (and
// every row of a bad utterance) get zeros and are not read.  CTCT: the flagged cells' occupancy is pb + pl + pr, and after
// the label terms above come - sum_q pr [k = y_u] (u >= 1), in increasing q.
constexpr int kGR = 64, kGC = 64, kGQ = 16;
template <int DT, bool GF, bool CTCT>
__device__ __forceinline__ void SimpleGrad(const void *f, const void *g, long long V, int Tmax, int Umax, const int *labels,
                                           int blank, const RnntMeta *meta, const float *mf, const float *mg, const int *ff,
                                           const int *fg, const float *S, const float *lse, const float *W, const float *PB,
                                           const float *PL, const float *PR, void *grad) {
    const int n = blockIdx.z;
    const RnntMeta m = meta[n];
    const int U1 = Umax + 1, Rmax = GF ? Tmax : U1;
    const int r0 = blockIdx.y * kGR;
    const long long c0 = (long long)blockIdx.x * kGC;
    const void *own = GF ? f : g, *oth = GF ? g : f;
    const float *m_own = GF ? mf : mg, *m_oth = GF ? mg : mf;
    const int *flag_own = GF ? ff : fg;
    const long long own0 = GF ? (long long)n * Tmax : (long long)n * U1, oth0 = GF ? (long long)n * U1 : (long long)n * Tmax;
    const long long fr0 = (long long)n * Tmax, gr0 = (long long)n * U1;
    const int Rn = m.bad ? 0 : (GF ? m.T : m.U + 1), Qn = m.bad ? 0 : (GF ? m.U + 1 : m.T);
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    // workspace row of cell (r, q)
    auto cell = [&](int r, int q) { return m.roff + (GF ? (long long)r * m.ts + q : (long long)q * m.ts + r); };
    float acc[4][4] = {};
    if (r0 < Rn) {
        __shared__ float As[kGQ][kGR + 1], Bs[kGQ][kGC];
        for (int q0 = 0; q0 < Qn; q0 += kGQ) {
#pragma unroll
            for (int i = 0; i < kGR * kGQ / 256; ++i) {
                const int e = tid + 256 * i, qq = e / kGR, rr = e % kGR, r = r0 + rr, q = q0 + qq;
                As[qq][rr] = r < Rn && q < Qn ? W[cell(r, q)] : 0.f;
            }
#pragma unroll
            for (int i = 0; i < kGC * kGQ / 256; ++i) {
                const int e = tid + 256 * i, qq = e / kGC, cc = e % kGC, q = q0 + qq;
                const long long k = c0 + cc;
                Bs[qq][cc] = q < Qn && k < V ? expf(load_y(oth, DT, (oth0 + q) * V + k) - SimpleOffset(m_oth[oth0 + q])) : 0.f;
            }
            __syncthreads();
#pragma unroll
            for (int qq = 0; qq < kGQ; ++qq) {
                float a[4], b[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) a[i] = As[qq][ty + 16 * i];
#pragma unroll
                for (int j = 0; j < 4; ++j) b[j] = Bs[qq][tx + 16 * j];
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
            }
            __syncthreads();
        }
    }
    // epilogue: acc becomes the gradient block
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int r = r0 + ty + 16 * i;
        if (r >= Rn) {
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
            continue;
        }
        const float mo = SimpleOffset(m_own[own0 + r]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const long long k = c0 + tx + 16 * j;
            acc[i][j] = k < V ? expf(load_y(own, DT, (own0 + r) * V + k) - mo) * acc[i][j] : 0.f;
        }
        if (flag_own[own0 + r]) {
            for (int q = 0; q < Qn; ++q) {
                const long long c = cell(r, q);
                if (!SimpleFlagged(S[c])) continue;
                const float occ = CTCT ? PB[c] + PL[c] + PR[c] : PB[c] + PL[c], Z = lse[c];
                const int t = GF ? r : q, u = GF ? q : r;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const long long k = c0 + tx + 16 * j;
                    if (k < V)
                        acc[i][j] += occ * expf(load_y(f, DT, (fr0 + t) * V + k) + load_y(g, DT, (gr0 + u) * V + k) - Z);
                }
            }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (c0 + tx + 16 * j != blank) continue;
            float sb = 0.f;
            for (int q = 0; q < Qn; ++q) sb += PB[cell(r, q)];
            acc[i][j] -= sb;
        }
        if (!GF && r < m.U) {      // grad_g: row u carries label y_{u+1}
            const int y = labels[m.loff + r];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (c0 + tx + 16 * j != y) continue;
                float sl = 0.f;
                for (int q = 0; q < Qn; ++q) sl += PL[cell(r, q)];
                acc[i][j] -= sl;
            }
        }
        if constexpr (CTCT) {
            if (!GF && r > 0) {    // grad_g: row u also carries the repeat of y_u
                const int y = labels[m.loff + r - 1];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    if (c0 + tx + 16 * j != y) continue;
                    float sr = 0.f;
                    for (int q = 0; q < Qn; ++q) sr += PR[cell(r, q)];
                    acc[i][j] -= sr;
                }
            }
        }
    }
    if (GF && r0 < Rn) {           // grad_f: label y_{u+1} of every u < U_n, in increasing u
        for (int q = 0; q < m.U; ++q) {
            const int y = labels[m.loff + q];
            const long long j = y - c0 - tx;
            if (j < 0 || j >= 16 * 4 || j % 16) continue;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int r = r0 + ty + 16 * i;
                if (r < Rn) {
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj)
                        if (jj == j / 16) acc[i][jj] -= PL[cell(r, q)];
                }
            }
        }
        if constexpr (CTCT) {      // then the repeat of y_u of every u >= 1, in increasing u
            for (int q = 1; q <= m.U; ++q) {
                const int y = labels[m.loff + q - 1];
                const long long j = y - c0 - tx;
                if (j < 0 || j >= 16 * 4 || j % 16) continue;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int r = r0 + ty + 16 * i;
                    if (r < Rn) {
#pragma unroll
                        for (int jj = 0; jj < 4; ++jj)
                            if (jj == j / 16) acc[i][jj] -= PR[cell(r, q)];
                    }
                }
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int r = r0 + ty + 16 * i;
        if (r >= Rmax) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const long long k = c0 + tx + 16 * j;
            if (k < V) store_y(grad, DT, (own0 + r) * V + k, acc[i][j]);
        }
    }
}

// GF before DT: the --profile reports of tools/*_bench.py key kernels by their first 60 characters, which then still
// tell grad_f from grad_g
template <bool CTCT, bool GF, int DT>
__global__ void __launch_bounds__(256) simple_grad_kernel(const void *f, const void *g, long long V, int Tmax, int Umax,
                                                          const int *labels, int blank, const RnntMeta *meta, const float *mf,
                                                          const float *mg, const int *ff, const int *fg, const float *S,
                                                          const float *lse, const float *W, const float *PB, const float *PL,
                                                          const float *PR, void *grad) {
    SimpleGrad<DT, GF, CTCT>(f, g, V, Tmax, Umax, labels, blank, meta, mf, mg, ff, fg, S, lse, W, PB, PL, PR, grad);
}

int GridX(long long rows_per_utt, int per_cta) {
    long long g = (rows_per_utt + per_cta - 1) / per_cta;
    return (int)std::max(1LL, std::min(g, 65535LL));
}

template <typename F>
void DispatchDtype(int dtype, F f) {
    if (dtype == CCB_DTYPE_F32) f(std::integral_constant<int, CCB_DTYPE_F32>{});
    else if (dtype == CCB_DTYPE_BF16) f(std::integral_constant<int, CCB_DTYPE_BF16>{});
    else f(std::integral_constant<int, CCB_DTYPE_F16>{});
}

bool RowsVectorisable(const void *p, long long V, int dtype) {
    const long long bytes = V * (dtype == CCB_DTYPE_F32 ? 4 : 2);
    return bytes % 16 == 0 && reinterpret_cast<uintptr_t>(p) % 16 == 0;
}

}  // namespace

template <bool CTCT> size_t TransducerLoss<CTCT>::WsBytes(int N, long long rows) {
    return MakeRnntLayout(N, rows, CTCT).total;
}

template <bool CTCT>
int TransducerLoss<CTCT>::Forward(const void *x, int dtype, int from_logits, int compact, int N, long long rows, int V, int Tmax,
                                  int Umax, const int *labels, long long n_labels, const int *lx, const int *ly, int blank,
                                  int want_beta, void *ws, float *costs, float *costs_beta, cudaStream_t s) {
    const RnntLayout L = MakeRnntLayout(N, rows, CTCT);
    RnntMeta *meta = At<RnntMeta>(ws, L.meta);
    float *lpb = At<float>(ws, L.lpb), *lpl = At<float>(ws, L.lpl), *lpr = AtOpt<float>(ws, L.lpr);
    rnnt_prep_kernel<<<1, kPrepThreads, 0, s>>>(lx, ly, N, rows, n_labels, compact, Tmax, Umax, meta, At<long long>(ws, L.tail));
    const long long per_utt = (rows + N - 1) / N;
    if (from_logits) {
        const int gx = GridX(per_utt, kRowThreads / 32 * 4);
        const bool vec = RowsVectorisable(x, V, dtype);
        DispatchDtype(dtype, [&](auto dt) {
            constexpr int DT = decltype(dt)::value;
            auto k = vec ? logit_rows_kernel<CTCT, DT, true> : logit_rows_kernel<CTCT, DT, false>;
            k<<<dim3(gx, N), kRowThreads, 0, s>>>(x, V, labels, blank, meta, lpb, lpl, lpr, At<float>(ws, L.lse));
        });
    } else {
        lp_rows_kernel<CTCT><<<dim3(GridX(per_utt, kRowThreads * 4), N), kRowThreads, 0, s>>>(x, dtype, V, labels, blank, meta,
                                                                                            lpb, lpl, lpr);
    }
    const auto alpha_beta = CTCT ? ctct_alpha_beta_kernel : rnnt_alpha_beta_kernel;
    alpha_beta<<<dim3(N, want_beta ? 2 : 1), kAbThreads, 0, s>>>(meta, labels, lpb, lpl, lpr, At<double>(ws, L.alpha),
                                                                 At<double>(ws, L.beta), At<double>(ws, L.logp), N, costs,
                                                                 want_beta ? costs_beta : nullptr);
    CountLaunch(3);
    return (int)cudaGetLastError();
}

template <bool CTCT>
int TransducerLoss<CTCT>::Backward(const void *x, int dtype, int from_logits, int N, long long rows, int V, const int *labels,
                                   int blank, void *ws, const float *w, void *grad, cudaStream_t s) {
    const RnntLayout L = MakeRnntLayout(N, rows, CTCT);
    const long long per_utt = (rows + N - 1) / N;
    const int gx = GridX(per_utt, kRowThreads / 32 * 4);
    const bool vec = RowsVectorisable(grad, V, dtype) && (!from_logits || RowsVectorisable(x, V, dtype));
    DispatchDtype(dtype, [&](auto dt) {
        constexpr int DT = decltype(dt)::value;
        auto k = from_logits ? (vec ? GradKernel<CTCT, DT, true, true>() : GradKernel<CTCT, DT, false, true>())
                             : (vec ? GradKernel<CTCT, DT, true, false>() : GradKernel<CTCT, DT, false, false>());
        k<<<dim3(gx, N + 1), kRowThreads, 0, s>>>(x, V, labels, blank, N, At<RnntMeta>(ws, L.meta), At<long long>(ws, L.tail),
                                                  rows, At<double>(ws, L.alpha), At<double>(ws, L.beta),
                                                  At<double>(ws, L.logp), At<float>(ws, L.lpb), At<float>(ws, L.lpl),
                                                  AtOpt<float>(ws, L.lpr), At<float>(ws, L.lse), w, grad);
    });
    CountLaunch(1);
    return (int)cudaGetLastError();
}

template <bool CTCT> size_t TransducerLoss<CTCT>::SimpleWsBytes(int N, int Tmax, int Umax) {
    return MakeSimpleLayout(N, Tmax, Umax, CTCT).total;
}

template <bool CTCT>
int TransducerLoss<CTCT>::SimpleForward(const void *f, const void *g, int dtype, int N, int Tmax, int Umax, int V,
                                        const int *labels, const int *lx, const int *ly, int blank, int want_beta, void *ws,
                                        float *costs, cudaStream_t s) {
    const SimpleLayout L = MakeSimpleLayout(N, Tmax, Umax, CTCT);
    const int U1 = Umax + 1;
    const long long cells = (long long)N * Tmax * U1;
    RnntMeta *meta = At<RnntMeta>(ws, L.r.meta);
    float *mf = At<float>(ws, L.mf), *mg = At<float>(ws, L.mg), *S = At<float>(ws, L.S);
    float *lpb = At<float>(ws, L.r.lpb), *lpl = At<float>(ws, L.r.lpl), *lpr = AtOpt<float>(ws, L.r.lpr);
    float *lse = At<float>(ws, L.r.lse);
    int *ff = At<int>(ws, L.ff), *fg = At<int>(ws, L.fg);
    rnnt_prep_kernel<<<1, kPrepThreads, 0, s>>>(lx, ly, N, cells, (long long)N * Umax, 0, Tmax, Umax, meta,
                                                At<long long>(ws, L.r.tail));
    const bool vec = RowsVectorisable(f, V, dtype) && RowsVectorisable(g, V, dtype);
    DispatchDtype(dtype, [&](auto dt) {
        constexpr int DT = decltype(dt)::value;
        auto rowmax = vec ? simple_rowmax_kernel<DT, true> : simple_rowmax_kernel<DT, false>;
        rowmax<<<dim3(GridX(std::max(Tmax, U1), kRowThreads / 32 * 4), N, 2), kRowThreads, 0, s>>>(f, g, V, Tmax, Umax, meta,
                                                                                                    mf, mg, ff, fg);
        simple_norm_kernel<CTCT, DT><<<dim3((Tmax + kST - 1) / kST, (U1 + kSU - 1) / kSU, N), 256, 0, s>>>(
            f, g, V, Tmax, Umax, labels, blank, meta, mf, mg, ff, fg, S, lpb, lpl, lpr, lse);
        auto fixup = vec ? simple_fixup_kernel<CTCT, DT, true> : simple_fixup_kernel<CTCT, DT, false>;
        fixup<<<dim3(GridX((long long)Tmax * U1, kRowThreads / 32 * 16), N), kRowThreads, 0, s>>>(
            f, g, V, Tmax, Umax, labels, blank, meta, ff, S, lpb, lpl, lpr, lse);
    });
    const auto alpha_beta = CTCT ? ctct_alpha_beta_kernel : rnnt_alpha_beta_kernel;
    alpha_beta<<<dim3(N, want_beta ? 2 : 1), kAbThreads, 0, s>>>(meta, labels, lpb, lpl, lpr, At<double>(ws, L.r.alpha),
                                                                 At<double>(ws, L.r.beta), At<double>(ws, L.r.logp), N, costs,
                                                                 nullptr);
    CountLaunch(5);
    return (int)cudaGetLastError();
}

template <bool CTCT>
int TransducerLoss<CTCT>::SimpleBackward(const void *f, const void *g, int dtype, int N, int Tmax, int Umax, int V,
                                         const int *labels, int blank, void *ws, const float *w, void *grad_f, void *grad_g,
                                         cudaStream_t s) {
    const SimpleLayout L = MakeSimpleLayout(N, Tmax, Umax, CTCT);
    const int U1 = Umax + 1;
    const RnntMeta *meta = At<RnntMeta>(ws, L.r.meta);
    const float *mf = At<float>(ws, L.mf), *mg = At<float>(ws, L.mg), *S = At<float>(ws, L.S), *lse = At<float>(ws, L.r.lse);
    const int *ff = At<int>(ws, L.ff), *fg = At<int>(ws, L.fg);
    float *W = At<float>(ws, L.W), *PB = At<float>(ws, L.PB), *PL = At<float>(ws, L.PL), *PR = AtOpt<float>(ws, L.PR);
    const auto weights = CTCT ? ctct_simple_weights_kernel : simple_weights_kernel;
    weights<<<dim3(GridX((long long)Tmax * U1, kRowThreads * 4), N), kRowThreads, 0, s>>>(
        meta, labels, At<double>(ws, L.r.alpha), At<double>(ws, L.r.beta), At<double>(ws, L.r.logp), At<float>(ws, L.r.lpb),
        At<float>(ws, L.r.lpl), AtOpt<float>(ws, L.r.lpr), S, w, W, PB, PL, PR);
    const int gx = (int)((V + kGC - 1) / kGC);
    DispatchDtype(dtype, [&](auto dt) {
        constexpr int DT = decltype(dt)::value;
        simple_grad_kernel<CTCT, true, DT><<<dim3(gx, (Tmax + kGR - 1) / kGR, N), 256, 0, s>>>(
            f, g, V, Tmax, Umax, labels, blank, meta, mf, mg, ff, fg, S, lse, W, PB, PL, PR, grad_f);
        simple_grad_kernel<CTCT, false, DT><<<dim3(gx, (U1 + kGR - 1) / kGR, N), 256, 0, s>>>(
            f, g, V, Tmax, Umax, labels, blank, meta, mf, mg, ff, fg, S, lse, W, PB, PL, PR, grad_g);
    });
    CountLaunch(3);
    return (int)cudaGetLastError();
}

template struct TransducerLoss<false>;
template struct TransducerLoss<true>;

size_t GatherWsBytes(int N) { return Align256(sizeof(GatherMeta) * (size_t)N); }

int LaunchGatherSum(const void *a, const void *b, int dtype, int N, long long rows_out, int H, const int *la, const int *lb,
                    void *ws, void *out, cudaStream_t s) {
    GatherMeta *meta = reinterpret_cast<GatherMeta *>(ws);
    gather_prep_kernel<<<1, kPrepThreads, 0, s>>>(la, lb, N, meta);
    const int gx = GridX((rows_out + N - 1) / N, kRowThreads / 32 * 4);
    DispatchDtype(dtype, [&](auto dt) {
        gather_sum_kernel<decltype(dt)::value><<<dim3(gx, N), kRowThreads, 0, s>>>(a, b, H, meta, out);
    });
    CountLaunch(2);
    return (int)cudaGetLastError();
}

int LaunchGatherSumBackward(const void *g, int dtype, int N, long long rows_a, long long rows_b, int H, const int *la,
                            const int *lb, void *ws, void *grad_a, void *grad_b, cudaStream_t s) {
    GatherMeta *meta = reinterpret_cast<GatherMeta *>(ws);
    gather_prep_kernel<<<1, kPrepThreads, 0, s>>>(la, lb, N, meta);
    DispatchDtype(dtype, [&](auto dt) {
        constexpr int DT = decltype(dt)::value;
        const int ga = GridX((rows_a + N - 1) / N, 1), gb = GridX((rows_b + N - 1) / N, 1);
        gather_sum_bwd_kernel<DT><<<dim3(ga, N), kRowThreads, 0, s>>>(g, H, meta, true, grad_a);
        gather_sum_bwd_kernel<DT><<<dim3(gb, N), kRowThreads, 0, s>>>(g, H, meta, false, grad_b);
    });
    CountLaunch(3);
    return (int)cudaGetLastError();
}

}  // namespace ccb
