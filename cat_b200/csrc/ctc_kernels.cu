// Numerator: per-utterance CTC forward-backward over the blank-expanded label lattice (log domain).
//
// Replaces src/ctc_crf/gpu_ctc (compute_alpha_kernel gpu_ctc_kernels.h:87-213,
// compute_betas_and_grad_kernel :218-458, host driver gpu_ctc.h:100-400).  Differences by design:
//   * nothing here touches the host (the reference synchronises the stream twice, gpu_ctc.h:272,368).  Each utterance
//     gets TWO CTAs in one launch: one walks alpha forwards while the other walks beta backwards at the same time
//     (both recursions are latency-bound chains of T frames, so this halves the critical path), each spilling its
//     cells relative to a per-frame fp64 offset; a second, fully parallel kernel (one warp per frame, all SMs) turns
//     the two spills into occupancies;
//   * thread i owns lattice cells 2i (blank) and 2i+1 (label i): the 2-/3-way log-sum of a frame needs
//     one value from the neighbouring thread, exchanged through a shared-memory ping-pong, one
//     __syncthreads per frame; the label row y[n][t][:] is staged coalesced one frame ahead;
//   * occupancies are reduced per label with shared-memory float atomics in the LINEAR domain (blank cells
//     are first summed with warp shuffles) -- no sort, no segmented reduce, no moderngpu;
//   * any layout: element (n,t,k) at n*sn + t*st + k, so the (N,T,V) logits are read in place (the
//     reference needs a transposed (T,N,V) copy, ctc_crf/__init__.py:70) and the gradient is ACCUMULATED
//     with a caller scale into a buffer that may already hold the denominator part;
//   * no 2L+1 <= 1280 limit (gpu_ctc.h:294-311): cells beyond the thread count are looped.
// Semantics kept: inputs are log-softmax outputs (gpu_ctc/README.txt:1-2); costs = log p(l|x);
// grad[t][k] = exp(LSE_{s: l'_s=k}(alpha_t(s)+beta_t(s)) - y_t(k) - log p) written for labels occurring in the
// utterance and t < len only (:431-435); infeasible utterances (L+repeats > T, :108-109) get
// log p = -inf and no gradient (the reference leaves both unwritten).
#include "common.cuh"

namespace ccb {

namespace {

constexpr unsigned kFull = 0xffffffffu;

// Precision: lattice cells are carried in DOUBLE, the log-add's transcendental part in float:
//     log_add(a, b[, c]) = m + (double) log(sum_i exp((float)(x_i - m))),   m = max_i x_i
// The float part is a number in [0, ln 3] with ~2e-7 absolute error whatever the magnitude of the cells, and the double
// sum does not quantise.  fp32 cells (round 1, relative to a per-frame offset) were not enough: at the cells that carry
// the occupancy mass, alpha lies ~ln C(t, t/2) - ln C(t, t/6) ~ 700 nats below the frame's alpha maximum at t = 3000
// (most alpha mass sits on paths that are ahead of the alignment), so |a_rel| ~ 700, ulp = 6e-5 per frame, and the
// occupancies came out 1.3e-3 (GPU) / 5e-3 (numpy float32 emulation) off the fp64 oracle at T = 3000.  With double cells
// the emulation gives 4e-7 at T = 3000.  (the reference's plain fp32 log domain: ~1e-2 at T ~ 1000.)
// Latency: a frame of the recursion is ONE dependent chain per thread (barrier -> neighbours' cells -> log-add -> cell), T of
// them in a row, so the chain length is the kernel's run time.  The 3-way log-sum of a label cell is therefore evaluated with
// one logarithm over the sum of the three exponentials (not two nested 2-way log-adds), and the exponentials / logarithm are
// the hardware ex2 / lg2 approximations: their arguments are differences to the maximum (|x| small, sum in [1, 3]), where
// they are as accurate in ABSOLUTE terms (ex2: 2 ulp of a number <= 1; lg2: 2^-22) as the libm versions.
// per-utterance workspace: alpha [T][ScMax] | beta [T][ScMax] doubles, then log p
__device__ __forceinline__ double log_add_d(double a, double b) {
    const double m = fmax(a, b);
    if (m == -INFINITY) return m;
    const float d = (float)(fmin(a, b) - m);          // <= 0; -inf when one side is empty: exp -> 0, log 1 -> 0
    return m + (double)__logf(1.f + __expf(d));
}
// c may be -inf ("no skip transition"): its exponential is then 0
__device__ __forceinline__ double log_add3_d(double a, double b, double c) {
    const double m = fmax(fmax(a, b), c);
    if (m == -INFINITY) return m;
    const float s = __expf((float)(a - m)) + __expf((float)(b - m)) + __expf((float)(c - m));   // one term is exp(0) = 1
    return m + (double)__logf(s);
}

struct CtcWorkspace {
    double *a = nullptr, *b = nullptr, *logp = nullptr;
    __device__ CtcWorkspace() {}
    __device__ CtcWorkspace(float *base, int n, int T, int ScMax) {
        const size_t cells = (size_t)T * ScMax;
        double *p = reinterpret_cast<double *>(base) + (size_t)n * (2 * cells + 1);
        a = p;
        b = p + cells;
        logp = p + 2 * cells;
    }
};

// shared memory carve-up: a[2][ScMax] doubles | lab[Lmax+1] ints | yrow[2][V] floats
// SPILL = false (forward-only loss): one CTA per utterance walks the alpha chain and writes only logp_out; no cell, no
// workspace.  The arithmetic is the same, so logp_out is bit-identical to the spilling launch's.
template <bool SPILL>
__global__ void ctc_alpha_beta_kernel(const void *y, int y_dtype, long sn, long st, int T, int V,
                                      const int *labels, const int *label_off, const int *label_len, const int *len,
                                      int max_label_len, int blank, float *alpha_ws, bool want_beta, float *logp_out,
                                      const double *lnorm) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int n = SPILL ? blockIdx.x >> 1 : blockIdx.x;
    const unsigned role = SPILL ? blockIdx.x & 1 : 0;   // 0: alpha pass, 1: beta pass
    const int tid = threadIdx.x, NT = blockDim.x;
    const int L = label_len[n], Tn = len[n];
    const int Sc = 2 * L + 1, L1 = L + 1;
    const int ScMax = 2 * max_label_len + 1;
    double *s_a = reinterpret_cast<double *>(smem_raw);                        // [2][ScMax]
    int *s_lab = reinterpret_cast<int *>(s_a + 2 * ScMax);                     // [max_label_len + 1] label of cell 2i+1
    float *s_y = reinterpret_cast<float *>(s_lab + max_label_len + 1);         // [2][V]
    const CtcWorkspace W = SPILL ? CtcWorkspace(alpha_ws, n, T, ScMax) : CtcWorkspace();
    const int *lab = labels + label_off[n];

    // feasibility (gpu_ctc_kernels.h:108-109)
    int rep = 0;
    for (int i = tid + 1; i < L; i += NT) rep += (lab[i] == lab[i - 1]);
    __shared__ int s_rep;
    if (tid == 0) s_rep = 0;
    __syncthreads();
    if (rep) atomicAdd(&s_rep, rep);
    __syncthreads();
    if (Tn <= 0 || L + s_rep > Tn) {
        if (tid == 0 && role == 0) { logp_out[n] = -INFINITY; if (SPILL) *W.logp = -INFINITY; }
        return;
    }
    if (!want_beta && role == 1) return;   // likelihood only
    for (int i = tid; i < L; i += NT) s_lab[i] = lab[i];
    double *ws = W.a, *wsb = W.b;
    const long ybase = n * sn;
    constexpr int kRowRegs = 4;
    const bool row_in_regs = V <= kRowRegs * NT;
    float yreg[kRowRegs];

    if (role == 0) {
    // ---- forward ---------------------------------------------------------------------------------
    for (int k = tid; k < V; k += NT) s_y[k] = load_y(y, y_dtype, ybase + k);
    __syncthreads();
    for (int s = tid; s < Sc; s += NT) {
        double v = -INFINITY;
        if (s == 0) v = (double)s_y[blank];
        else if (s == 1) v = (double)s_y[s_lab[0]];
        s_a[s] = v;
        if (SPILL) ws[s] = v;
    }
    // Row prefetch: the emission row of frame t+1 is loaded into registers while frame t is computed and parked in
    // shared memory afterwards, so no frame waits on a global-memory round trip (V <= kRowRegs * blockDim).
    if (row_in_regs && Tn > 1) {
#pragma unroll
        for (int j = 0; j < kRowRegs; ++j) { const int k = tid + j * NT; yreg[j] = k < V ? load_y(y, y_dtype, ybase + st + k) : 0.f; }
#pragma unroll
        for (int j = 0; j < kRowRegs; ++j) { const int k = tid + j * NT; if (k < V) s_y[V + k] = yreg[j]; }
    }
    for (int t = 1; t < Tn; ++t) {
        // One barrier per frame: it publishes row t (parked in slot t&1 during the previous frame) and the previous cells.
        float *yc = s_y + (t & 1) * V;
        const double *prev = s_a + ((t - 1) & 1) * ScMax;
        double *cur = s_a + (t & 1) * ScMax;
        if (!row_in_regs) for (int k = tid; k < V; k += NT) yc[k] = load_y(y, y_dtype, ybase + (long)t * st + k);
        else if (t + 1 < Tn) {
#pragma unroll
            for (int j = 0; j < kRowRegs; ++j) { const int k = tid + j * NT; yreg[j] = k < V ? load_y(y, y_dtype, ybase + (long)(t + 1) * st + k) : 0.f; }
        }
        __syncthreads();
        for (int i = tid; i < L1; i += NT) {
            // blank cell 2i
            const int sb = 2 * i;
            double vb = prev[sb];
            if (i > 0) vb = log_add_d(vb, prev[sb - 1]);
            vb += (double)yc[blank];
            cur[sb] = vb;
            if (SPILL) ws[(size_t)t * ScMax + sb] = vb;
            if (i < L) {   // label cell 2i+1
                const int sl = sb + 1;
                const int li = s_lab[i];
                const bool skip = i > 0 && li != s_lab[i - 1];
                double vl = log_add3_d(prev[sl], prev[sb], skip ? prev[sl - 2] : -INFINITY);
                vl += (double)yc[li];
                cur[sl] = vl;
                if (SPILL) ws[(size_t)t * ScMax + sl] = vl;
            }
        }
        if (row_in_regs && t + 1 < Tn) {   // park row t+1 in the slot last read during frame t-1
            float *yn = s_y + ((t + 1) & 1) * V;
#pragma unroll
            for (int j = 0; j < kRowRegs; ++j) { const int k = tid + j * NT; if (k < V) yn[k] = yreg[j]; }
        }
    }
    __syncthreads();
    if (tid == 0) {
        const double *last = s_a + ((Tn - 1) & 1) * ScMax;
        double lp = last[Sc - 1];
        if (Sc > 1) lp = log_add_d(lp, last[Sc - 2]);
        // raw-logit entry: the reported log-likelihood is normalised; everything else stays in the raw domain
        logp_out[n] = (float)(lp - (lnorm ? lnorm[n] : 0.0));
        if (SPILL) *W.logp = lp;
    }
    } else if (SPILL) {
    // ---- beta pass (the utterance's second CTA), concurrent with the alpha pass -------------------------
    {
        const int t = Tn - 1;
        float *yc = s_y + (t & 1) * V;
        for (int k = tid; k < V; k += NT) yc[k] = load_y(y, y_dtype, ybase + (long)t * st + k);
    }
    for (int t = Tn - 1; t >= 0; --t) {
        float *yc = s_y + (t & 1) * V;
        double *cur = s_a + (t & 1) * ScMax;
        const double *nxt = s_a + ((t + 1) & 1) * ScMax;
        if (t > 0 && row_in_regs) {   // issue the loads for frame t-1 now; they are parked after this frame's work
#pragma unroll
            for (int j = 0; j < kRowRegs; ++j) { const int k = tid + j * NT; yreg[j] = k < V ? load_y(y, y_dtype, ybase + (long)(t - 1) * st + k) : 0.f; }
        }
        __syncthreads();   // the only barrier of the frame: publishes row t and beta_{t+1}
        double *bl = wsb + (size_t)t * ScMax;
        for (int i = tid; i < L1; i += NT) {
            const int sb = 2 * i;
            double vb;
            if (t == Tn - 1) {
                vb = (sb == Sc - 1) ? (double)yc[blank] : -INFINITY;
            } else {
                vb = nxt[sb];
                if (sb + 1 < Sc) vb = log_add_d(vb, nxt[sb + 1]);
                vb += (double)yc[blank];
            }
            cur[sb] = vb;
            bl[sb] = vb;
            if (i < L) {
                const int sl = sb + 1;
                const int li = s_lab[i];
                double vl;
                if (t == Tn - 1) {
                    vl = (sl == Sc - 2) ? (double)yc[li] : -INFINITY;
                } else {
                    const bool skip = i + 1 < L && li != s_lab[i + 1];
                    vl = log_add3_d(nxt[sl], nxt[sl + 1], skip ? nxt[sl + 2] : -INFINITY);
                    vl += (double)yc[li];
                }
                cur[sl] = vl;
                bl[sl] = vl;
            }
        }
        if (t > 0) {   // park row t-1 in the slot last read during frame t+1
            float *yn = s_y + ((t - 1) & 1) * V;
            if (row_in_regs) {
#pragma unroll
                for (int j = 0; j < kRowRegs; ++j) { const int k = tid + j * NT; if (k < V) yn[k] = yreg[j]; }
            } else {
                for (int k = tid; k < V; k += NT) yn[k] = load_y(y, y_dtype, ybase + (long)(t - 1) * st + k);
            }
        }
    }
    }

}

// Occupancies from the two spills: one warp per (utterance, frame), label accumulator [V] per warp in shared memory.
//   gamma_t[k] = sum_{s: l'_s = k} exp(alpha_t(s) + beta_t(s) - y_t(k) - log p)   (gpu_ctc_kernels.h:337-453)
// accumulated with the caller's scale into grad[n][t][:] (which may already hold the denominator part).
// zero_inf: this is the first launch after both halves of the loss, so it is where an utterance whose cost is not finite
// (log p, or logz[n] when the den part is given, not finite) is masked: its rows t < len[n] are written with zeros, den
// part included, instead of accumulated.
__global__ void ctc_gamma_kernel(const void *y, int y_dtype, long sn, long st, int N, int T, int V,
                                 const int *labels, const int *label_off, const int *label_len, const int *len,
                                 int max_label_len, int blank, float *alpha_ws,
                                 float *grad, long gsn, long gst, float grad_scale, int overwrite, int Tfull,
                                 const float *logz, int zero_inf) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    const long row = (long)blockIdx.x * wpb + warp;
    // overwrite mode (CTC-only loss): every row of the (N, Tfull, V) gradient is WRITTEN, zeros included, so the caller
    // needs no zero-fill pass; accumulate mode adds into a buffer that already holds the denominator part.
    const int Trows = overwrite ? Tfull : T;
    if (row >= (long)N * Trows) return;
    const int n = (int)(row / Trows), t = (int)(row % Trows);
    const int L = label_len[n], Sc = 2 * L + 1, ScMax = 2 * max_label_len + 1;
    CtcWorkspace W(alpha_ws, n, T, ScMax);
    const double logp_d = *W.logp;
    const bool masked = zero_inf && !(isfinite(logp_d) && (logz == nullptr || isfinite(logz[n])));
    if (t >= len[n] || masked || !(logp_d > -INFINITY)) {      // padding frame / infeasible or masked utterance: no gradient
        if (overwrite || (masked && t < len[n])) {
            float *gz = grad + n * gsn + (long)t * gst;
            for (int k = lane; k < V; k += 32) gz[k] = 0.f;
        }
        return;
    }
    float *g = reinterpret_cast<float *>(smem_raw) + (size_t)warp * V;
    for (int k = lane; k < V; k += 32) g[k] = 0.f;
    __syncwarp();
    const double *al = W.a + (size_t)t * ScMax, *bl = W.b + (size_t)t * ScMax;
    const int *lab = labels + label_off[n];
    const long yrow = n * sn + (long)t * st;
    float occ_blank = 0.f;
    for (int s = lane; s < Sc; s += 32) {   // lane parity == cell parity: even lanes take blanks, odd lanes labels
        const int li = (s & 1) ? __ldg(lab + (s >> 1)) : blank;
        const float o = (float)(al[s] + bl[s] - (double)load_y(y, y_dtype, yrow + li) - logp_d);
        const float e = (o == -INFINITY || o != o) ? 0.f : expf(o);
        if (s & 1) { if (e != 0.f) atomicAdd(&g[li], e); }
        else occ_blank += e;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) occ_blank += __shfl_xor_sync(kFull, occ_blank, o);
    __syncwarp();
    if (lane == 0 && occ_blank != 0.f) g[blank] += occ_blank;
    __syncwarp();
    float *grow = grad + n * gsn + (long)t * gst;
    for (int k = lane; k < V; k += 32) {
        const float gv = g[k];
        if (overwrite) grow[k] = grad_scale * gv;
        else if (gv != 0.f) atomicAdd(grow + k, grad_scale * gv);
    }
}

// cost[n] = -logp[n];  loss[0] = scale * sum_n cost[n]   (CTC-only loss, ctc_crf/__init__.py:41-47: costs = -sum log p, / batch
// when averaging).  costs (optional) receives each cost; zero_inf sets a cost that is not finite to 0 first.
__global__ void sum_scale_kernel(const float *logp, int N, float scale, float *loss, float *costs, int zero_inf) {
    double acc = 0.0;
    for (int n = threadIdx.x; n < N; n += 32) {
        double c = -(double)logp[n];
        if (zero_inf && !isfinite(c)) c = 0.0;
        if (costs) costs[n] = (float)c;
        acc += c;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(kFull, acc, o);
    if (threadIdx.x == 0) loss[0] = (float)(acc * (double)scale);
}

// out[n][t][:] = w[n] * grad[n][t][:], converted to out_dtype, one warp per row; rows t >= len[n] are written with zeros
// without reading grad.  The per-utterance weighted backward of a loss with reduction 'none'.
__global__ void grad_rows_scale_kernel(const float *grad, const float *w, const int *len, int N, int T, int V, void *out,
                                       int out_dtype) {
    const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
    const long row = (long)blockIdx.x * wpb + (threadIdx.x >> 5);
    if (row >= (long)N * T) return;
    const int n = (int)(row / T), t = (int)(row % T);
    const long base = row * V;
    if (t >= len[n]) {
        for (int k = lane; k < V; k += 32) store_y(out, out_dtype, base + k, 0.f);
        return;
    }
    const float wn = __ldg(w + n);
    for (int k = lane; k < V; k += 32) store_y(out, out_dtype, base + k, wn * __ldg(grad + base + k));
}

// Best-path (Viterbi) alignment over the same blank-expanded lattice: the forced alignment that is a by-product of the
// numerator (SURVEY 8f-4).  One CTA per utterance; thread i owns cells 2i and 2i+1 as in the alpha pass; max replaces
// log-add; a 2-bit back-pointer per cell and frame (0: stay, 1: from s-1, 2: from s-2) goes to the workspace, and thread 0
// walks it back.  align[n][t] = the token emitted at frame t (blank included), -1 for t >= len or an utterance without a
// path of finite score (too few frames for its labels, or every path through a -inf emission).
// Ties are broken towards the smaller predecessor index (stay < s-1 < s-2).
// shared memory: lab[Lmax] ints | v[2][ScMax] floats
__global__ void ctc_viterbi_kernel(const void *y, int y_dtype, long sn, long st, int T, int V,
                                   const int *labels, const int *label_off, const int *label_len, const int *len,
                                   int max_label_len, int blank, unsigned char *bp_ws, int *align, float *score) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int n = blockIdx.x, tid = threadIdx.x, NT = blockDim.x;
    const int L = label_len[n], Tn = len[n];
    const int Sc = 2 * L + 1, L1 = L + 1, ScMax = 2 * max_label_len + 1;
    int *s_lab = reinterpret_cast<int *>(smem_raw);
    float *s_v = reinterpret_cast<float *>(s_lab + max_label_len + 1);
    unsigned char *bp = bp_ws + (size_t)n * T * ScMax;
    const int *lab = labels + label_off[n];
    int *arow = align + (size_t)n * T;
    for (int t = tid; t < T; t += NT) arow[t] = -1;
    int rep = 0;
    for (int i = tid + 1; i < L; i += NT) rep += (lab[i] == lab[i - 1]);
    __shared__ int s_rep;
    if (tid == 0) s_rep = 0;
    __syncthreads();
    if (rep) atomicAdd(&s_rep, rep);
    __syncthreads();
    if (Tn <= 0 || L + s_rep > Tn) { if (tid == 0 && score) score[n] = -INFINITY; return; }
    for (int i = tid; i < L; i += NT) s_lab[i] = lab[i];
    __syncthreads();
    const long ybase = n * sn;
    for (int s = tid; s < Sc; s += NT) {
        float v = -INFINITY;
        if (s == 0) v = load_y(y, y_dtype, ybase + blank);
        else if (s == 1) v = load_y(y, y_dtype, ybase + s_lab[0]);
        s_v[s] = v;
        bp[s] = 0;
    }
    for (int t = 1; t < Tn; ++t) {
        __syncthreads();
        const float *prev = s_v + ((t - 1) & 1) * ScMax;
        float *cur = s_v + (t & 1) * ScMax;
        unsigned char *b = bp + (size_t)t * ScMax;
        const long yrow = ybase + (long)t * st;
        for (int i = tid; i < L1; i += NT) {
            const int sb = 2 * i;
            float vb = prev[sb];
            unsigned char kb = 0;
            if (i > 0 && prev[sb - 1] > vb) { vb = prev[sb - 1]; kb = 1; }
            cur[sb] = vb + load_y(y, y_dtype, yrow + blank);
            b[sb] = kb;
            if (i < L) {
                const int sl = sb + 1, li = s_lab[i];
                float vl = prev[sl];
                unsigned char kl = 0;
                if (prev[sb] > vl) { vl = prev[sb]; kl = 1; }
                if (i > 0 && li != s_lab[i - 1] && prev[sl - 2] > vl) { vl = prev[sl - 2]; kl = 2; }
                cur[sl] = vl + load_y(y, y_dtype, yrow + li);
                b[sl] = kl;
            }
        }
    }
    __syncthreads();
    if (tid == 0) {
        const float *last = s_v + ((Tn - 1) & 1) * ScMax;
        int s = Sc - 1;
        if (Sc > 1 && last[Sc - 2] > last[Sc - 1]) s = Sc - 2;
        if (score) score[n] = last[s];
        // every path killed by -inf emissions: the back-pointers lead nowhere, so the row keeps its -1s
        if (last[s] == -INFINITY) return;
        for (int t = Tn - 1; t >= 0; --t) {
            arow[t] = (s & 1) ? s_lab[s >> 1] : blank;
            s -= bp[(size_t)t * ScMax + s];
        }
    }
}

// cost[n] = logz[n] - (1+lamb) logp[n];  loss[0] = scale * sum_n cost[n]      (ctc_crf/__init__.py:79-86)
// costs (optional) receives each cost; zero_inf sets a cost that is not finite to 0 first.
__global__ void assemble_loss_kernel(const float *logz, const float *logp, int N, float lamb, float scale, float *loss,
                                     float *costs, int zero_inf) {
    double acc = 0.0;
    for (int n = threadIdx.x; n < N; n += 32) {
        double c = (double)logz[n] - (1.0 + (double)lamb) * (double)logp[n];
        if (zero_inf && !isfinite(c)) c = 0.0;
        if (costs) costs[n] = (float)c;
        acc += c;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(kFull, acc, o);
    if (threadIdx.x == 0) loss[0] = (float)(acc * (double)scale);
}

// The two halves of the numerator: the alpha || beta chains write the cell workspace + logp, the occupancy kernel turns
// the cells into the gradient.  alpha_ws = null: the forward-only launch (the alpha chains alone, logp only).
int LaunchCtcAlphaBeta(const void *y, int y_dtype, long sn, long st, int N, int T, int V, const int *labels,
                       const int *label_off, const int *label_len, const int *len, int max_label_len, int blank,
                       float *alpha_ws, bool want_beta, float *logp, const double *lnorm, cudaStream_t stream,
                       std::string *err) {
    if (N == 0) return 0;
    const int ScMax = 2 * max_label_len + 1;
    int threads = ((max_label_len + 1 + 31) / 32) * 32;
    threads = threads < 64 ? 64 : (threads > 1024 ? 1024 : threads);
    // two emission rows of V floats are staged in shared memory, so V bounds the vocabulary: at most 25 505 classes with
    // label sequences of up to 20 (the lattice rows take 16 * (2 Lmax + 1) + 4 * (Lmax + 1) + 16 bytes of the 200 KB)
    constexpr size_t kSmemLimit = 200 * 1024;
    const size_t lattice = (size_t)2 * ScMax * 8 + (size_t)(max_label_len + 1) * 4 + 16;
    const size_t smem = lattice + (size_t)2 * V * 4;
    if (smem > kSmemLimit) {
        const long v_max = lattice < kSmemLimit ? (long)((kSmemLimit - lattice) / 8) : 0;
        *err = "numerator kernel: V = " + std::to_string(V) + " classes with label sequences of up to " +
               std::to_string(max_label_len) + " need " + std::to_string(smem) + " bytes of shared memory (two emission rows " +
               "of V floats plus the lattice), above its limit of " + std::to_string(kSmemLimit) + " bytes; at this label " +
               "length V may be at most " + std::to_string(v_max);
        return 1;
    }
    const bool spill = alpha_ws != nullptr;
    const void *kernel = spill ? (const void *)ctc_alpha_beta_kernel<true> : (const void *)ctc_alpha_beta_kernel<false>;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { *err = std::string("cudaFuncSetAttribute(ctc): ") + cudaGetErrorString(e); return (int)e; }
    if (spill)
        ctc_alpha_beta_kernel<true><<<2 * N, threads, smem, stream>>>(y, y_dtype, sn, st, T, V, labels, label_off, label_len, len,
                                                                      max_label_len, blank, alpha_ws, want_beta, logp, lnorm);
    else
        ctc_alpha_beta_kernel<false><<<N, threads, smem, stream>>>(y, y_dtype, sn, st, T, V, labels, label_off, label_len, len,
                                                                   max_label_len, blank, nullptr, false, logp, lnorm);
    CountLaunch();
    e = cudaGetLastError();
    if (e != cudaSuccess) { *err = std::string("ctc launch: ") + cudaGetErrorString(e); return (int)e; }
    return 0;
}

int LaunchCtcGamma(const void *y, int y_dtype, long sn, long st, int N, int T, int V, const int *labels,
                   const int *label_off, const int *label_len, const int *len, int max_label_len, int blank,
                   float *alpha_ws, float *grad, long gsn, long gst, float grad_scale, cudaStream_t stream,
                   std::string *err, int overwrite, int Tfull, const float *logz, int zero_inf) {
    if (N == 0) return 0;
    int wpb = 8;   // warps (= frames) per CTA of the occupancy kernel, bounded by the [V] accumulators
    while (wpb > 1 && (size_t)wpb * V * 4 > 48 * 1024) wpb >>= 1;
    const size_t gsm = (size_t)wpb * V * 4;
    cudaError_t e = cudaFuncSetAttribute(ctc_gamma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gsm);
    if (e != cudaSuccess) { *err = std::string("cudaFuncSetAttribute(ctc gamma): ") + cudaGetErrorString(e); return (int)e; }
    const long rows = (long)N * (overwrite ? Tfull : T);
    ctc_gamma_kernel<<<(unsigned)((rows + wpb - 1) / wpb), wpb * 32, gsm, stream>>>(
        y, y_dtype, sn, st, N, T, V, labels, label_off, label_len, len, max_label_len, blank, alpha_ws, grad, gsn, gst, grad_scale,
        overwrite, Tfull, logz, zero_inf);
    CountLaunch();
    e = cudaGetLastError();
    if (e != cudaSuccess) { *err = std::string("ctc gamma launch: ") + cudaGetErrorString(e); return (int)e; }
    return 0;
}

}  // namespace

int LaunchCtc(const void *y, int y_dtype, long sn, long st, int N, int T, int V, const int *labels,
              const int *label_off, const int *label_len, const int *len, int max_label_len, int blank,
              float *alpha_ws, float *grad, long gsn, long gst, float grad_scale, float *logp,
              const double *lnorm, cudaStream_t stream, std::string *err, int overwrite, int Tfull, const float *logz,
              int zero_inf) {
    int rc = LaunchCtcAlphaBeta(y, y_dtype, sn, st, N, T, V, labels, label_off, label_len, len, max_label_len, blank, alpha_ws,
                                grad != nullptr, logp, lnorm, stream, err);
    if (rc || grad == nullptr) return rc;
    return LaunchCtcGamma(y, y_dtype, sn, st, N, T, V, labels, label_off, label_len, len, max_label_len, blank, alpha_ws, grad, gsn,
                          gst, grad_scale, stream, err, overwrite, Tfull, logz, zero_inf);
}

int LaunchCtcLogp(const void *y, int y_dtype, long sn, long st, int N, int T, int V, const int *labels,
                  const int *label_off, const int *label_len, const int *len, int max_label_len, int blank, float *logp,
                  const double *lnorm, cudaStream_t stream, std::string *err) {
    return LaunchCtcAlphaBeta(y, y_dtype, sn, st, N, T, V, labels, label_off, label_len, len, max_label_len, blank, nullptr,
                              false, logp, lnorm, stream, err);
}

int LaunchSumScale(const float *logp, int N, float scale, float *loss, cudaStream_t stream, float *costs, int zero_inf) {
    sum_scale_kernel<<<1, 32, 0, stream>>>(logp, N, scale, loss, costs, zero_inf);
    CountLaunch();
    return (int)cudaGetLastError();
}

int LaunchGradRowsScale(const float *grad, const float *w, const int *len, int N, int T, int V, void *out, int out_dtype,
                        cudaStream_t stream) {
    const long rows = (long)N * T;
    if (rows == 0) return 0;
    const int wpb = 8;
    grad_rows_scale_kernel<<<(unsigned)((rows + wpb - 1) / wpb), wpb * 32, 0, stream>>>(grad, w, len, N, T, V, out, out_dtype);
    CountLaunch();
    return (int)cudaGetLastError();
}

int LaunchCtcViterbi(const void *y, int y_dtype, long sn, long st, int N, int T, int V, const int *labels,
                     const int *label_off, const int *label_len, const int *len, int max_label_len, int blank,
                     unsigned char *bp_ws, int *align, float *score, cudaStream_t stream, std::string *err) {
    if (N == 0) return 0;
    const int ScMax = 2 * max_label_len + 1;
    int threads = ((max_label_len + 1 + 31) / 32) * 32;
    threads = threads < 64 ? 64 : (threads > 1024 ? 1024 : threads);
    const size_t smem = (size_t)(max_label_len + 1) * 4 + (size_t)2 * ScMax * 4;
    if (smem > 200 * 1024) { *err = "label sequence too long for the alignment kernel's shared memory"; return 1; }
    cudaError_t e = cudaFuncSetAttribute(ctc_viterbi_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { *err = std::string("cudaFuncSetAttribute(ctc viterbi): ") + cudaGetErrorString(e); return (int)e; }
    ctc_viterbi_kernel<<<N, threads, smem, stream>>>(y, y_dtype, sn, st, T, V, labels, label_off, label_len, len, max_label_len,
                                                     blank, bp_ws, align, score);
    CountLaunch();
    e = cudaGetLastError();
    if (e != cudaSuccess) { *err = std::string("ctc viterbi launch: ") + cudaGetErrorString(e); return (int)e; }
    return 0;
}

int LaunchAssembleLoss(const float *logz, const float *logp, int N, float lamb, float scale, float *loss,
                       cudaStream_t stream, float *costs, int zero_inf) {
    assemble_loss_kernel<<<1, 32, 0, stream>>>(logz, logp, N, lamb, scale, loss, costs, zero_inf);
    CountLaunch();
    return (int)cudaGetLastError();
}

}  // namespace ccb
