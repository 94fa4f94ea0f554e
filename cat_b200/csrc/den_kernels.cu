// Denominator forward-backward over the shared phone-LM WFST: persistent sm_90a kernels.
//
// What the reference does (src/ctc_crf/gpu_den/den_calculate.cu): 3T+6 launches of <<<N,1024>>> kernels,
// one CTA per utterance, thread per state, log-domain log1p(exp()) per arc, per-arc atomicCAS gradient.
//
// What this file does instead (DESIGN.md "Denominator"):
//   * batched sparse semiring SpMM: lanes = utterances, a warp walks the arcs of its rows; every arc is
//     one coalesced row gather alpha[t-1][peer][n0..n0+U) from L2 + U FMAs.  Arc metadata is read once
//     per 32*U utterances and lives in shared memory for the whole kernel (loaded once per launch).
//   * scaled-linear arithmetic: alpha/beta are kept in the linear domain with a per-(frame,utterance)
//     power-of-two scale (exact), so the arc loop has no transcendental at all; the emission
//     exp(y - max_k y) is applied once per (state, frame) thanks to the loader's single-in-label states.
//   * one cooperative launch per pass; frames are separated by a hand-rolled grid barrier
//     (red.release arrive, relaxed polling, one acquire fence), not by kernel launches.
//   * gradient without arc atomics: gamma_t[k] = sum_{q: lab(q)=k} alpha_t(q) beta_t(q) / sum_q alpha_t(q) beta_t(q),
//     accumulated per CTA in shared memory (states are sorted by label) and flushed with a few REDs.
#include <cstdio>
#include <cstdlib>

#include "common.cuh"

namespace ccb {

namespace {

// Per-frame column sums are renormalised to ~2^E with E = DenParams::scale_exp (56 unless the graph's out-weight sums are
// large, den_graph.cc): the scale a frame is written with comes from the PREVIOUS column, so a frame whose emissions are all
// tiny (one-hot rows with -60 floors cost 2^-87) sits that far below 2^E for one frame; values live down to 2^-149, which
// leaves 2^-(E+149) / drop of dynamic range inside such a column.  E = 32 lost 6e-2 on the occupancies there (measured,
// tests/test_gpu_atsize.py::test_peaky_logits), E >= 48 is exact to 4e-6; the ceiling is the occupancy product
// alpha * beta <= 2^(2E+2) * G^2 < 2^127 (G = largest out-weight sum of a state).
constexpr unsigned kFull = 0xffffffffu;

// Row gathers read data that another SM wrote one frame earlier.  Plain (L1-allocating) loads are coherent here: every
// frame ends in the grid barrier's gpu-scope acquire fence + bar.sync, after which ordinary loads must observe the other
// CTAs' released writes (the same contract cooperative-groups grid.sync() gives), and no row is re-read within a frame
// after being rewritten.  Against ld.global.cg this makes the zero-weight padding slots (which repeat the address of
// the preceding arc) L1 hits.
template <int U> struct Vec;
template <> struct Vec<1> {
    float v[1];
    __device__ __forceinline__ static Vec ld_row(const float *p) { Vec r; r.v[0] = *p; return r; }
    __device__ __forceinline__ void stcg(float *p) const { __stcg(p, v[0]); }
};
template <> struct Vec<2> {
    float v[2];
    __device__ __forceinline__ static Vec ld_row(const float *p) {
        float2 t = *reinterpret_cast<const float2 *>(p);
        Vec r; r.v[0] = t.x; r.v[1] = t.y; return r;
    }
    __device__ __forceinline__ void stcg(float *p) const { __stcg(reinterpret_cast<float2 *>(p), make_float2(v[0], v[1])); }
};
template <> struct Vec<4> {
    float v[4];
    __device__ __forceinline__ static Vec ld_row(const float *p) {
        float4 t = *reinterpret_cast<const float4 *>(p);
        Vec r; r.v[0] = t.x; r.v[1] = t.y; r.v[2] = t.z; r.v[3] = t.w; return r;
    }
    __device__ __forceinline__ void stcg(float *p) const {
        __stcg(reinterpret_cast<float4 *>(p), make_float4(v[0], v[1], v[2], v[3]));
    }
};
template <int U> __device__ __forceinline__ Vec<U> vec_zero() {
    Vec<U> r;
#pragma unroll
    for (int u = 0; u < U; ++u) r.v[u] = 0.f;
    return r;
}

// r = 2^shift with shift = E - floor(log2(s)); exact power of two, so rescaling never rounds.
__device__ __forceinline__ float scale_from_sum(float s, int *shift, int E) {
    if (!(s > 0.f) || s > 3.0e38f) { *shift = 0; return 1.f; }
    int field = (__float_as_int(s) >> 23) & 0xff;
    int ex = (field == 0 ? 1 : field) - 127;
    int sh = E - ex;
    sh = max(-126, min(127, sh));
    *shift = sh;
    return __int_as_float((sh + 127) << 23);
}

// One quad of arcs as two 16-byte words: {peer0..3} and {w0..3}.  In shared memory the tile is staged quad-wise in
// exactly this (SoA) form, so each word is one LDS.128 whose four lanes are all used; the global-memory fallback
// (tiles too large for shared memory) reads the plan's AoS arcs.
// forward gather rows: peers >= S name virtual pair-sum rows, parked at 2S + j of the frame (see den_forward_kernel)
__device__ __forceinline__ uint32_t fwd_row(uint32_t peer, int S) { return peer < (uint32_t)S ? peer : peer + (uint32_t)S; }
// virt_from: peers >= virt_from are shifted by virt_from (forward pass: S; backward pass: no virtual rows, 0xffffffff)
template <bool SMEM_ARCS>
__device__ __forceinline__ uint4 load_quad_peers(const uint4 *quad, uint32_t row_bytes, uint32_t virt_from = 0xffffffffu) {
    if (SMEM_ARCS) return quad[0];   // already byte offsets
    const uint4 m0 = __ldg(quad), m1 = __ldg(quad + 1);
    auto row = [&](uint32_t p) { return (p >= virt_from ? p + virt_from : p) * row_bytes; };
    return make_uint4(row(m0.x), row(m0.z), row(m1.x), row(m1.z));
}
template <bool SMEM_ARCS>
__device__ __forceinline__ uint4 load_quad_weights(const uint4 *quad) {
    if (SMEM_ARCS) return quad[1];
    const uint4 m0 = __ldg(quad), m1 = __ldg(quad + 1);
    return make_uint4(m0.y, m0.w, m1.y, m1.w);
}

// Row address = 64-bit lane base + 32-bit BYTE offset (two integer adds; ptxas splits every mad.wide form into three
// instructions, so the multiplication by the row pitch is done once, when the tile is staged / in the fallback loader).
template <int U>
__device__ __forceinline__ Vec<U> gather_row(const char *lane_base, uint32_t byte_off) {
    return Vec<U>::ld_row(reinterpret_cast<const float *>(lane_base + byte_off));
}
// The gathers of one quad.  (Skipping the zero-weight padding slots -- ~17 % of the forward stream -- with a per-quad
// count in the last offset costs more in branches than the saved gathers return.)
template <int U>
__device__ __forceinline__ void gather_quad(const char *lane_base, const uint4 pr, Vec<U> *v) {
    v[0] = gather_row<U>(lane_base, pr.x);
    v[1] = gather_row<U>(lane_base, pr.y);
    v[2] = gather_row<U>(lane_base, pr.z);
    v[3] = gather_row<U>(lane_base, pr.w);
}
template <int U>
__device__ __forceinline__ float *row_ptr(float *lane_base, uint32_t row, uint32_t row_bytes) {
    return reinterpret_cast<float *>(reinterpret_cast<char *>(lane_base) + (size_t)row * row_bytes);
}

__device__ __forceinline__ void prefetch_l2(const void *p) {
    asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}

// ------------------------------------------------------------------------------------------------
// per-frame emission shift  m[t][n] = max_k y[n][t][k]
// ------------------------------------------------------------------------------------------------
__global__ void frame_max_kernel(const void *y, int dtype, long sn, long st, int N, int T, int V,
                                 const int *len, float *fmax, int Npad) {
    const int warps_per_block = blockDim.x >> 5;
    const long row = (long)blockIdx.x * warps_per_block + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= (long)N * T) return;
    const int n = (int)(row / T), t = (int)(row % T);
    if (t >= len[n]) return;
    float m = -INFINITY;
    const long base = n * sn + t * st;
    for (int k = lane; k < V; k += 32) m = fmaxf(m, load_y(y, dtype, base + k));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(kFull, m, o));
    if (lane == 0) fmax[(size_t)t * Npad + n] = (m == -INFINITY) ? 0.f : m;
}

// Raw-logit entry (SURVEY 8f-1): per valid frame the max AND the log-normaliser lz = log sum_k exp(z_k) of the raw
// encoder outputs.  The recursions then run on z as if it were log-probs (emissions are shifted by the row max either
// way, and a per-frame constant does not change any occupancy); only the log-likelihoods need lz, summed per utterance.
__global__ void frame_lse_kernel(const void *y, int dtype, long sn, long st, int N, int T, int V,
                                 const int *len, float *fmax, float *lz, int Npad) {
    const int warps_per_block = blockDim.x >> 5;
    const long row = (long)blockIdx.x * warps_per_block + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= (long)N * T) return;
    const int n = (int)(row / T), t = (int)(row % T);
    if (t >= len[n]) return;
    float m = -INFINITY;
    const long base = n * sn + t * st;
    for (int k = lane; k < V; k += 32) m = fmaxf(m, load_y(y, dtype, base + k));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(kFull, m, o));
    if (m == -INFINITY) m = 0.f;
    float s = 0.f;
    for (int k = lane; k < V; k += 32) s += expf(load_y(y, dtype, base + k) - m);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(kFull, s, o);
    if (lane == 0) {
        fmax[(size_t)t * Npad + n] = m;
        lz[(size_t)t * Npad + n] = m + logf(s);
    }
}

// lnorm[n] = sum_{t < len[n]} lz[t][n] in fp64, fixed order (one warp per utterance)
__global__ void lnorm_kernel(const float *lz, const int *len, int N, int Npad, double *lnorm) {
    const int n = blockIdx.x, lane = threadIdx.x;
    double acc = 0.0;
    const int ln = len[n];
    for (int t = lane; t < ln; t += 32) acc += (double)lz[(size_t)t * Npad + n];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(kFull, acc, o);
    if (lane == 0) lnorm[n] = acc;
}

// Softmax Jacobian of the raw-logit entry: g = dL/dy (y = log_softmax z) -> dL/dz_k = g_k - softmax(z)_k * sum_j g_j,
// in place, one warp per valid frame (cat/ctc/train.py:173-174 does this through autograd of log_softmax).
__global__ void logit_grad_kernel(const void *z, int dtype, long sn, long st, int N, int T, int V, const int *len,
                                  const float *lz, int Npad, float *grad, long gsn, long gst) {
    const int warps_per_block = blockDim.x >> 5;
    const long row = (long)blockIdx.x * warps_per_block + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= (long)N * T) return;
    const int n = (int)(row / T), t = (int)(row % T);
    if (t >= len[n]) return;
    float *g = grad + n * gsn + t * gst;
    float gs = 0.f;
    for (int k = lane; k < V; k += 32) gs += g[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) gs += __shfl_xor_sync(kFull, gs, o);
    // a row whose entries sum to 0 loses nothing; skipping it keeps a zeroed row (zero_infinity) zero where the frame's
    // logits are all -inf and expf(z - lz) = expf(-inf + inf) is NaN
    if (gs == 0.f) return;
    const float l = lz[(size_t)t * Npad + n];
    const long base = n * sn + t * st;
    for (int k = lane; k < V; k += 32) g[k] -= expf(load_y(z, dtype, base + k) - l) * gs;
}

// ------------------------------------------------------------------------------------------------
// The arc walk shared by both passes: a software-pipelined stream over the warp's chunk of arcs.
//   * arcs come a quad at a time: one LDS.128 of four peers for the gathers, one LDS.128 of four weights for the FMAs;
//   * BATCH row gathers (plain loads, 32*U*4 bytes each, one per arc) are issued for batch k+1 BEFORE batch k
//     is consumed, so a warp keeps BATCH..2*BATCH loads in flight (the recursion is latency-bound on L2);
//   * weights are applied as |w|; the sign bit of a quad's 4th weight marks the end of a segment and the sign bits
//     of its 3rd/2nd weights the event code (den_graph.h kEv*): `seg_end(acc, event)` runs (warp-uniform branch).
// `arcs` points at the chunk's first quad (two 16-byte words per quad), n_batches = chunk arcs / BATCH.
// ------------------------------------------------------------------------------------------------
template <int U, int BATCH, bool SMEM_ARCS, typename Prologue, typename SegEnd>
__device__ __forceinline__ void walk_arcs(const uint4 *arcs, int n_batches, uint32_t row_bytes, uint32_t virt_from, const char *lane_base,
                                          bool do_load, Prologue &&prologue, SegEnd &&seg_end) {
    Vec<U> vA[BATCH], vB[BATCH];
#pragma unroll
    for (int i = 0; i < BATCH; ++i) { vA[i] = vec_zero<U>(); vB[i] = vec_zero<U>(); }   // lanes that never load stay 0
    float acc[U];
#pragma unroll
    for (int u = 0; u < U; ++u) acc[u] = 0.f;

    // issue: arc words are transient here (only the offsets are needed); consume re-reads them from shared memory
    // for the weights, which keeps 2*BATCH gathers in flight without holding 2*BATCH arc words in registers.
    // a quad is two 16-byte words (peers, weights); `issue` needs only the first, `consume` only the second, so
    // 2*BATCH gathers stay in flight without holding 2*BATCH arc words in registers.
    auto issue = [&](const uint4 *p, Vec<U> *v) {
        if (do_load) {
            // all offset words first: the per-quad padding branch below must not sit between a quad's shared-memory
            // load and the next one (that exposed the LDS latency once per quad)
            uint4 pr[BATCH / kQuad];
#pragma unroll
            for (int g4 = 0; g4 < BATCH / kQuad; ++g4) pr[g4] = load_quad_peers<SMEM_ARCS>(p + 2 * g4, row_bytes, virt_from);
#pragma unroll
            for (int g4 = 0; g4 < BATCH / kQuad; ++g4) gather_quad<U>(lane_base, pr[g4], v + g4 * kQuad);
        }
    };
    auto consume = [&](const uint4 *p, const Vec<U> *v) {
#pragma unroll
        for (int g4 = 0; g4 < BATCH / kQuad; ++g4) {
            const uint4 wq = load_quad_weights<SMEM_ARCS>(p + 2 * g4);
            const float w0 = fabsf(__uint_as_float(wq.x)), w1 = fabsf(__uint_as_float(wq.y));
            const float w2 = fabsf(__uint_as_float(wq.z)), w3 = fabsf(__uint_as_float(wq.w));
            float a2[U];   // the sums WITHOUT the quad's last slot (kEvPairMerged: that slot belongs to the pair's other row)
#pragma unroll
            for (int u = 0; u < U; ++u) {
                acc[u] = fmaf(w0, v[g4 * kQuad + 0].v[u], acc[u]);
                acc[u] = fmaf(w1, v[g4 * kQuad + 1].v[u], acc[u]);
                acc[u] = fmaf(w2, v[g4 * kQuad + 2].v[u], acc[u]);
                a2[u] = acc[u];
                acc[u] = fmaf(w3, v[g4 * kQuad + 3].v[u], acc[u]);
            }
            if ((int)wq.w < 0)   // warp-uniform: a segment ends at this quad; the callback owns the accumulators
                seg_end(acc, (int)(((wq.z >> 31) << 1) | (wq.y >> 31)), (int)wq.x < 0, p + 2 * g4, a2, v[g4 * kQuad + 3], w3);
        }
    };

    const uint4 *pi = arcs, *pc = arcs;
    int nb = n_batches;   // batches not yet consumed
    if (nb <= 0) { prologue(); return; }
    issue(pi, vA); pi += BATCH / 2;
    if (nb > 1) { issue(pi, vB); pi += BATCH / 2; }
    prologue();   // per-frame scalars (scales, emissions) are fetched while the first gathers are in flight
    while (true) {
        consume(pc, vA); pc += BATCH / 2;
        if (--nb == 0) break;
        if (nb > 1) { issue(pi, vA); pi += BATCH / 2; }
        consume(pc, vB); pc += BATCH / 2;
        if (--nb == 0) break;
        if (nb > 1) { issue(pi, vB); pi += BATCH / 2; }
    }
}

// Backward variant: every slot carries two weights (den_graph.h DenPlan::bwd) -- w0 for the group's first row, w1 for
// its second row -- so the arcs shared by the two members of a pair are gathered once and feed two accumulators.
// Shared-memory quads are three 16-byte words {byte offsets}{w0}{w1}; the global fallback reads the plan's AoS arcs
// plus the separate w1 array.  `group_end(acc0, acc1, pair, new_label0, new_label1)` runs at the last quad of a group.
// W1_SMEM = false with SMEM_ARCS = true is the middle tier for graphs whose 12-byte backward slots do not fit shared
// memory: byte offsets and first weights stay in shared memory (8 bytes per slot), the second weights stream from L2.
template <int U, int BATCH, bool SMEM_ARCS, bool W1_SMEM, typename Prologue, typename GroupEnd>
__device__ __forceinline__ void walk_arcs_dual(const uint4 *arcs, const float4 *w1g, int n_batches, uint32_t row_bytes,
                                               const char *lane_base, bool do_load, Prologue &&prologue, GroupEnd &&group_end) {
    constexpr int kWordsPerQuad = (SMEM_ARCS && W1_SMEM) ? 3 : 2;
    // middle tier, one utterance per lane (the registers allow it): the second weights of a batch are fetched from L2
    // together with its gathers instead of at consume time
    constexpr bool kPrefW1 = SMEM_ARCS && !W1_SMEM && U == 1;
    constexpr int kQ = BATCH / kQuad;
    Vec<U> vA[BATCH], vB[BATCH];
    float4 wA[kPrefW1 ? kQ : 1], wB[kPrefW1 ? kQ : 1];
#pragma unroll
    for (int i = 0; i < BATCH; ++i) { vA[i] = vec_zero<U>(); vB[i] = vec_zero<U>(); }
#pragma unroll
    for (int i = 0; i < (kPrefW1 ? kQ : 1); ++i) { wA[i] = make_float4(0.f, 0.f, 0.f, 0.f); wB[i] = wA[i]; }
    float acc0[U], acc1[U];
#pragma unroll
    for (int u = 0; u < U; ++u) { acc0[u] = 0.f; acc1[u] = 0.f; }

    auto issue = [&](const uint4 *p, const float4 *pw1, Vec<U> *v, float4 *wpre) {
        if (do_load) {
            if (kPrefW1) {
#pragma unroll
                for (int g4 = 0; g4 < kQ; ++g4) wpre[g4] = __ldg(pw1 + g4);
            }
            uint4 pr[BATCH / kQuad];
#pragma unroll
            for (int g4 = 0; g4 < BATCH / kQuad; ++g4) pr[g4] = SMEM_ARCS ? p[kWordsPerQuad * g4] : load_quad_peers<false>(p + 2 * g4, row_bytes);
#pragma unroll
            for (int g4 = 0; g4 < BATCH / kQuad; ++g4) gather_quad<U>(lane_base, pr[g4], v + g4 * kQuad);
        }
    };
    auto consume = [&](const uint4 *p, const float4 *pw1, const Vec<U> *v, const float4 *wpre) {
#pragma unroll
        for (int g4 = 0; g4 < BATCH / kQuad; ++g4) {
            const uint4 wq = SMEM_ARCS ? p[kWordsPerQuad * g4 + 1] : load_quad_weights<false>(p + 2 * g4);
            float4 w1;
            if (kPrefW1) w1 = wpre[g4];
            else if (SMEM_ARCS && W1_SMEM) { const uint4 t = p[kWordsPerQuad * g4 + 2]; w1 = make_float4(__uint_as_float(t.x), __uint_as_float(t.y), __uint_as_float(t.z), __uint_as_float(t.w)); }
            else w1 = __ldg(pw1 + g4);
            const float a0 = fabsf(__uint_as_float(wq.x)), a1 = fabsf(__uint_as_float(wq.y));
            const float a2 = fabsf(__uint_as_float(wq.z)), a3 = fabsf(__uint_as_float(wq.w));
#pragma unroll
            for (int u = 0; u < U; ++u) {
                acc0[u] = fmaf(a0, v[g4 * kQuad + 0].v[u], acc0[u]);
                acc1[u] = fmaf(w1.x, v[g4 * kQuad + 0].v[u], acc1[u]);
                acc0[u] = fmaf(a1, v[g4 * kQuad + 1].v[u], acc0[u]);
                acc1[u] = fmaf(w1.y, v[g4 * kQuad + 1].v[u], acc1[u]);
                acc0[u] = fmaf(a2, v[g4 * kQuad + 2].v[u], acc0[u]);
                acc1[u] = fmaf(w1.z, v[g4 * kQuad + 2].v[u], acc1[u]);
                acc0[u] = fmaf(a3, v[g4 * kQuad + 3].v[u], acc0[u]);
                acc1[u] = fmaf(w1.w, v[g4 * kQuad + 3].v[u], acc1[u]);
            }
            if ((int)wq.w < 0)   // warp-uniform: the group ends at this quad
                group_end(acc0, acc1, (int)wq.z < 0, (int)wq.x < 0, (int)wq.y < 0);
        }
    };

    constexpr int kStep = kWordsPerQuad * (BATCH / kQuad);   // 16-byte words per batch
    const uint4 *pi = arcs, *pc = arcs;
    const float4 *pw = w1g, *pwi = w1g;
    int nb = n_batches;
    if (nb <= 0) { prologue(); return; }
    issue(pi, pwi, vA, wA); pi += kStep; pwi += kQ;
    if (nb > 1) { issue(pi, pwi, vB, wB); pi += kStep; pwi += kQ; }
    prologue();
    while (true) {
        consume(pc, pw, vA, wA); pc += kStep; pw += kQ;
        if (--nb == 0) break;
        if (nb > 1) { issue(pi, pwi, vA, wA); pi += kStep; pwi += kQ; }
        consume(pc, pw, vB, wB); pc += kStep; pw += kQ;
        if (--nb == 0) break;
        if (nb > 1) { issue(pi, pwi, vB, wB); pi += kStep; pwi += kQ; }
    }
}

// ------------------------------------------------------------------------------------------------
// TMA row gathers (sm_90a): one tile-mode `cp.async.bulk.tensor.2d` (a box of one row of the gather table) per arc slot,
// issued by the lanes of the warp, one row each.  The rows of a batch land in a per-warp ring (STAGES stages of R rows)
// and complete an mbarrier; the warp then reads them with LDS.  A row coordinate beyond the tensor (kOobRow) is
// zero-filled by the TMA unit without touching L2.  The rows in flight cost no registers.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, unsigned parity) {
    unsigned ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    } while (!ok);
}
// one row (the tensor map's box: 1 row x box_cols columns) into shared memory; `dst` must be 128-byte aligned
__device__ __forceinline__ void tma_row(uint32_t dst, const CUtensorMap *tm, int col, int row, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(dst), "l"(tm), "r"(col), "r"(row), "r"(bar) : "memory");
}
// the arc slot j (0..3) of a quad's row word
__device__ __forceinline__ int quad_row(const uint4 &pr, int j) { return (int)(j == 0 ? pr.x : j == 1 ? pr.y : j == 2 ? pr.z : pr.w); }
// 1-D bulk copy global -> shared (SASS UBLKCP): sequential arc words of a batch, completing on the batch's mbarrier
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, unsigned bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// rows written with ordinary stores by other CTAs are read through the async proxy (TMA) one frame later: order the two
// proxies on both sides of the grid barrier
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

// per-warp ring state: shared-memory address of the ring, of its first mbarrier, and the parity to wait for per stage
struct TmaRing {
    uint32_t buf, bar, phase;
};

template <int U> __device__ __forceinline__ Vec<U> lds_row(uint32_t addr);
template <> __device__ __forceinline__ Vec<1> lds_row<1>(uint32_t addr) {
    Vec<1> r;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(r.v[0]) : "r"(addr));
    return r;
}
template <> __device__ __forceinline__ Vec<2> lds_row<2>(uint32_t addr) {
    Vec<2> r;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(r.v[0]), "=f"(r.v[1]) : "r"(addr));
    return r;
}

// Streamed arcs (graphs whose arc stream does not fit shared memory, BASELINE config 4: 5 M arcs): the chunk's quads are
// not resident; they flow through a per-warp ring of kArcStages batches, filled by 1-D bulk copies (`cp.async.bulk`, SASS
// UBLKCP: the stream is sequential and the same every frame) from DevicePass::tq, each stage completing its own mbarrier.
// The ring is topped up after every consumed batch and runs across frames and lane groups: the first kArcStages batches
// of the NEXT walk are requested at the end of this one, so they are in shared memory before the grid barrier opens.
// Batches are counted from the start of the kernel (stage = count % kArcStages, parity = count / kArcStages & 1).
struct ArcRing {
    const uint4 *buf;        // this warp's ring in shared memory ...
    uint32_t buf_s, bar;     // ... its shared-memory address, and its first mbarrier
    uint32_t issued, done;   // batches requested / consumed so far
    uint32_t src_k, n;       // next batch of the chunk to request (wraps at n = batches per walk)
    const uint4 *src;        // the chunk's quads in global memory
};
template <int AW>   // AW = 16-byte words per batch
__device__ __forceinline__ void arc_ring_fill(ArcRing &ar, int lane) {
    if (ar.n == 0) return;
    while (ar.issued != ar.done + kArcStages) {
        if (lane == 0) {
            const uint32_t st = ar.issued % kArcStages, bar = ar.bar + 8u * st;
            mbar_expect_tx(bar, AW * 16u);
            bulk_g2s(ar.buf_s + st * (AW * 16u), ar.src + (size_t)ar.src_k * AW, AW * 16u, bar);
        }
        ++ar.issued;
        if (++ar.src_k == ar.n) ar.src_k = 0;
    }
}
// before the kernel ends: no bulk copy may still be in flight into this CTA's shared memory
__device__ __forceinline__ void arc_ring_drain(ArcRing &ar) {
    while (ar.done != ar.issued) {
        mbar_wait(ar.bar + 8u * (ar.done % kArcStages), (ar.done / kArcStages) & 1u);
        ++ar.done;
    }
}
// The arc walk with TMA-staged rows over the streamed quads (WPQ 16-byte words each, {row index 0..3}{w0..3}{w1 0..3}):
// n_batches = chunk arcs / R, one batch = R/4 quads whose rows lanes 0..R-1 request (one row each).  `consume_quad(words of
// the quad, rows v[4])` does the FMAs and the group-end work.
template <int U, int R, int WPQ, typename Prologue, typename ConsumeQuad>
__device__ __forceinline__ void walk_arcs_tma_stream(ArcRing &ar, int n_batches, const CUtensorMap *tm, int col, int row_base,
                                                     TmaRing &ring, int lane, Prologue &&prologue, ConsumeQuad &&consume_quad) {
    constexpr int QB = R / kQuad, AW = QB * WPQ;
    constexpr uint32_t ROWB = 32u * U * 4u;
    static_assert(R % kQuad == 0 && kChunkArcPad % R == 0 && R <= 32, "a batch is whole quads, divides the chunk padding, one row per lane");
    const uint32_t g0 = ar.done;
    auto issue = [&](int k, int s) {
        const uint32_t g = g0 + (uint32_t)k, st = g % kArcStages;
        mbar_wait(ar.bar + 8u * st, (g / kArcStages) & 1u);   // every lane: the batch's arc words have landed
        const uint32_t bar = ring.bar + 8u * s;
        if (lane == 0) mbar_expect_tx(bar, R * ROWB);
        __syncwarp();
        if (lane < R) {
            const uint4 pr = ar.buf[st * AW + WPQ * (lane / kQuad)];
            tma_row(ring.buf + (uint32_t)(s * R + lane) * ROWB, tm, col, row_base + quad_row(pr, lane % kQuad), bar);
        }
    };
    auto consume = [&](int k, int s) {
        mbar_wait(ring.bar + 8u * s, (ring.phase >> s) & 1u);
        ring.phase ^= 1u << s;
        const uint32_t base = ring.buf + (uint32_t)(s * R) * ROWB + (uint32_t)lane * (U * 4u);
        const uint4 *quads = ar.buf + ((g0 + (uint32_t)k) % kArcStages) * AW;
#pragma unroll
        for (int q = 0; q < QB; ++q) {
            Vec<U> v[kQuad];
#pragma unroll
            for (int j = 0; j < kQuad; ++j) v[j] = lds_row<U>(base + (uint32_t)(q * kQuad + j) * ROWB);
            consume_quad(quads + WPQ * q, v);
        }
        __syncwarp();   // every lane is done with the row stage and the arc stage before they are refilled
        ar.done = g0 + (uint32_t)k + 1u;
        arc_ring_fill<AW>(ar, lane);
    };
    if (n_batches <= 0) { prologue(); return; }
    issue(0, 0);
    if (n_batches > 1) issue(1, 1);
    prologue();
    for (int k = 0; k < n_batches; k += 2) {
        consume(k, 0);
        if (k + 2 < n_batches) issue(k + 2, 0);
        if (k + 1 < n_batches) {
            consume(k + 1, 1);
            if (k + 3 < n_batches) issue(k + 3, 1);
        }
    }
}

// Small batches (Npad = 16 utterances): a row of the gather table is 64 bytes, and the lanes of a warp are spread over (arc
// of the quad) x (utterance): the four rows of a quad lie back to back in the ring, so two `LDS.32` per lane read 2 arcs x
// 16 utterances each, each lane multiplies by the weight of ITS arc, and the two lane groups' partial sums are combined with
// one shuffle when a segment ends: half the instructions and rows of L2 traffic per utterance of 16 idle lanes (the per-GPU
// share of a batch sharded over 8 GPUs is 8-32 utterances, SURVEY.md 8e).  Rings: kSmallStages stages of kSmallRows rows
// per warp.  Rows this short sit below the 128-byte alignment a tensor copy's destination needs, so each row is a 1-D bulk
// copy from `table` (16-byte alignment), one per lane; the lane of a padding slot (kOobRow) zero-fills its row instead.
__device__ __forceinline__ float lds_f32(uint32_t addr) {
    float r;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(r) : "r"(addr));
    return r;
}
// W1_STREAM (backward pass of graphs whose 12-byte slots do not fit shared memory): the SECOND weights of a batch -- 16
// consecutive floats of DenPlan::bwd.w1 -- are not resident; they ride along with the batch's rows as one 64-byte bulk copy
// into `w1buf` (one 64-byte slot per stage) on the same mbarrier, and `consume_quad` receives their shared-memory address.
template <int WPQ, bool W1_STREAM = false, typename Prologue, typename ConsumeQuad>
__device__ __forceinline__ void walk_arcs_tma_small(const uint4 *arcs, int n_batches, const float *table, int row_base,
                                                    TmaRing &ring, int lane, Prologue &&prologue, ConsumeQuad &&consume_quad,
                                                    const float *w1g = nullptr, uint32_t w1buf = 0u) {
    constexpr int R = kSmallRows, QB = R / kQuad;
    constexpr uint32_t ROWB = kSmallLanes * 4u;
    auto issue = [&](int k, int s) {
        const uint32_t bar = ring.bar + 8u * s, dst = ring.buf + (uint32_t)(s * R + lane) * ROWB;
        const uint32_t row = lane < R ? (uint32_t)quad_row(arcs[(size_t)WPQ * (k * QB + lane / kQuad)], lane % kQuad) : kOobRow;
        const unsigned live = __ballot_sync(0xffffffffu, row != kOobRow);
        if (lane < R && row == kOobRow) {
#pragma unroll
            for (uint32_t b = 0; b < ROWB; b += 16u)
                asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(dst + b), "r"(0u) : "memory");
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // before a later bulk copy refills the slot
        }
        if (lane == 0) {
            mbar_expect_tx(bar, (unsigned)__popc(live) * ROWB + (W1_STREAM ? R * 4u : 0u));
            if (W1_STREAM) bulk_g2s(w1buf + 64u * s, w1g + (size_t)k * R, R * 4u, bar);
        }
        __syncwarp();   // (also orders the zero stores before every lane's reads of the stage)
        if (row != kOobRow) bulk_g2s(dst, table + (size_t)(row_base + (int)row) * kSmallLanes, ROWB, bar);
    };
    if (n_batches <= 0) { prologue(); return; }
    for (int k = 0; k < kSmallStages && k < n_batches; ++k) issue(k, k);
    prologue();
    for (int k = 0; k < n_batches; ++k) {
        const int s = k & (kSmallStages - 1);
        mbar_wait(ring.bar + 8u * s, (ring.phase >> s) & 1u);
        ring.phase ^= 1u << s;
        const uint32_t base = ring.buf + (uint32_t)(s * R) * ROWB + (uint32_t)lane * 4u;
#pragma unroll
        for (int q = 0; q < QB; ++q) {
            float v[2];   // slots sub and 2 + sub (two LDS steps per quad)
#pragma unroll
            for (int st = 0; st < 2; ++st) v[st] = lds_f32(base + (uint32_t)q * (kQuad * ROWB) + (uint32_t)st * 128u);
            consume_quad(arcs + (size_t)WPQ * (k * QB + q), v, w1buf + 64u * s + 16u * q);
        }
        __syncwarp();
        if (k + kSmallStages < n_batches) issue(k + kSmallStages, s);
    }
}
// weight of arc j (0..3) of a quad's weight word
__device__ __forceinline__ uint32_t quad_word(const uint4 &w, int j) { return j == 0 ? w.x : j == 1 ? w.y : j == 2 ? w.z : w.w; }

__device__ __forceinline__ unsigned long long global_timer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
// optional per-warp timeline (debug/profiling only): [step][chunk][4] = {globaltimer at step start,
// clock64 at step start, clock64 when the chunk is done, clock64 after the grid barrier}
__device__ __forceinline__ void tl_mark(const DenParams &P, int step_index, int chunk, int n_chunks, int slot, int lane) {
    if (P.timeline == nullptr || lane != 0) return;
    const int s = step_index - P.tl_step0;
    if (s < 0 || s >= P.tl_steps) return;
    unsigned long long *rec = P.timeline + ((size_t)s * n_chunks + chunk) * 4;
    if (slot == 0) { rec[0] = global_timer(); rec[1] = clock64(); }
    else rec[slot + 1] = clock64();
}

// One PART of a high in-degree forward row (den_graph.h kEvPartial): scale the partial sum like a row end and add it
// into the target row with atomics (the row was zeroed one frame ahead).  Deliberately out of line and self-contained:
// it recomputes the few per-frame scalars it needs so that the hot row-end path keeps its registers.
template <int U>
__device__ __noinline__ void forward_partial_row(const int *state_label, const int *len, const float *colsum_prev,
                                                 const float *fmax_prev, const void *y, int y_dtype, long sn, long yt_off,
                                                 int N, int t, int n0, Vec<U> part, uint32_t tgt_off, uint32_t row_bytes,
                                                 float *a_cur, float *s_sum, int scale_exp) {
    const int tgt = (int)(tgt_off / row_bytes);
    const int lab = __ldg(state_label + tgt);
    float *dst = reinterpret_cast<float *>(reinterpret_cast<char *>(a_cur + n0) + tgt_off);
#pragma unroll
    for (int u = 0; u < U; ++u) {
        const int n = n0 + u;
        if (n < N && t <= __ldg(len + n)) {
            int sh;
            const float r = scale_from_sum(__ldcg(colsum_prev + n), &sh, scale_exp);
            const float e = expf(load_y(y, y_dtype, n * sn + yt_off + lab) - __ldg(fmax_prev + n));
            const float o = part.v[u] * e * r;
            if (o != 0.f) { atomicAdd(dst + u, o); atomicAdd(&s_sum[n], o); }
        }
    }
}

// Position of alpha frame t in DenParams::alpha.  Full spill: t.  Recompute of a segment: t - a_base (frames a_base ..
// a_base + K, plus two for the parked rows of the last ones).  First checkpointed pass: t mod a_ring on a ring of
// a_ring = kAlphaRing positions followed by 2 slack positions.  The layout stays relative to the frame: frame t's pair-sum
// rows are parked at row 2S + j of ITS base, i.e. in position p + 2 (p = its position, so the slack when p >= a_ring - 2),
// and frame t's hub rows are zeroed during frame t - 1.  While frame t is computed the live positions are p(t-1) with its
// parked rows at p(t-1) + 2 (read), p(t) and p(t) + 2 (written) and p(t+1) (hub rows zeroed); four ring positions keep
// the writes off everything frame t reads (three would land frame t's parked rows on frame t-1 when p(t) = 0), and a
// position is rewritten a_ring frames later, after every reader of it has passed a grid barrier.
__device__ __forceinline__ int alpha_pos(const DenParams &P, int t) {
    const int p = t - P.a_base;
    return P.a_ring > 0 ? p % P.a_ring : p;
}

// First checkpointed pass, once frame t is complete (after its grid barrier): keep a copy of its real rows if it is a
// checkpoint, and add sum_q final(q) alpha_t(q, n) to zsum for the utterances that end at frame t (their frame is gone
// from the ring by the end of the pass).  (Inlined: a call in the frame loop would save its live registers around it.)
__device__ __forceinline__ void ckpt_frame_done(const DenParams &P, int t, const float *fr, int sb, int se, int lane) {
    const size_t frame_elems = (size_t)P.S * P.Npad;
    if (t % P.ckpt_k == 0 && t < P.Tmax) {   // (S * Npad is a multiple of 16 floats)
        const float4 *src = reinterpret_cast<const float4 *>(fr);
        float4 *dst = reinterpret_cast<float4 *>(P.ckpt + (size_t)(t / P.ckpt_k) * frame_elems);
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < frame_elems / 4; i += (size_t)gridDim.x * blockDim.x)
            __stcg(dst + i, __ldcg(src + i));
    }
    for (int gc = 0; gc < (P.Npad + 31) / 32; ++gc) {
        const int n = gc * 32 + lane;
        const bool ends = n < P.N && __ldg(P.len + n) == t;
        if (!__any_sync(kFull, ends)) continue;
        float zs = 0.f;
        if (ends) {
            for (int q = sb; q < se; ++q) {
                const float f = __ldg(P.final_lin + q);
                if (f != 0.f) zs = fmaf(f, __ldcg(fr + (size_t)q * P.Npad + n), zs);
            }
        }
        if (zs != 0.f) atomicAdd(P.zsum + n, zs);
    }
}

// ------------------------------------------------------------------------------------------------
// forward: alpha recursion + logZ
// ------------------------------------------------------------------------------------------------
// HUBS: the plan contains high in-degree rows split into parts (kEvPartial segments); the common case compiles the
// partial-row path out entirely so that it costs the hot row-end code nothing.
// Rows are gathered into registers (walk_arcs), except in the small-batch variant (SMALL: 16 lanes per row), whose rows
// are staged in shared memory by bulk copies (TMA, walk_arcs_tma_small); it needs the arc tile in shared memory
// (SMEM_ARCS), one utterance per lane and no hub rows.
template <int U, int BATCH, bool SMEM_ARCS, bool HUBS, bool SMALL = false>
__global__ void __launch_bounds__(kDenThreads, 1) den_forward_kernel(const __grid_constant__ DenParams P) {
    constexpr int LPR = SMALL ? kSmallLanes : 32;   // lanes per row
    static_assert(!SMALL || (SMEM_ARCS && U == 1 && !HUBS), "small-batch variant: arc tile in shared memory, one utterance per lane, no hubs");
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float *s_sum = reinterpret_cast<float *>(smem_raw);                                  // [Npad]
    int *s_label = reinterpret_cast<int *>(s_sum + P.Npad);                              // [tile_rows] label per row
    Arc *s_arcs = reinterpret_cast<Arc *>(smem_raw + FwdArcsOff(P.Npad, P.tile_rows));

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(kFull, tid >> 5, 0);   // (through a shuffle: lets ptxas keep warp-derived addresses in uniform registers)
    const int sub = LPR == 32 ? 0 : lane / LPR;    // small batches: which arc(s) of a quad this lane multiplies
    const int ul = LPR == 32 ? lane : lane % LPR;   // ... and which utterance(s) it carries
    const int cta = blockIdx.x;
    const int chunk = cta * P.n_warps + warp;
    const int n_chunks = gridDim.x * P.n_warps;
    const int sb = __ldg(P.chunk_state + chunk), se = __ldg(P.chunk_state + chunk + 1);
    const int ab = __ldg(P.chunk_arc + chunk), ae = __ldg(P.chunk_arc + chunk + 1);
    const int tile_a0 = __ldg(P.chunk_arc + cta * P.n_warps);
    const int tile_a1 = __ldg(P.chunk_arc + (cta + 1) * P.n_warps);
    const int tile_s0 = __ldg(P.chunk_state + cta * P.n_warps);
    const int tile_s1 = __ldg(P.chunk_state + (cta + 1) * P.n_warps);
    const int vj0 = __ldg(P.chunk_pair + chunk);   // first virtual (pair-sum) row written by this warp
    const int S = P.S, Npad = P.Npad;
    // Spill layout: frame t holds the S real rows only (what the backward pass reads back from HBM).  The virtual pair-sum
    // rows of frame t -- read by frame t+1 only -- are parked where the real rows of frame t+2 will be written: gather
    // peer S + j maps to row 2S + j of the frame, so one base pointer still addresses everything a frame gathers, the parked
    // rows are overwritten in L2 two frames later and never reach HBM, and the spill is (T+3) * S rows instead of
    // (T+1) * (S+P)  (N=64, T=1500, 1 M arcs: 15.4 GB instead of 23 GB; forward DRAM writes 10.2 MB instead of 15 MB a frame).
    const size_t frame_elems = (size_t)S * Npad;
    const uint32_t virt0 = 2u * (uint32_t)S;                       // first parked virtual row, relative to the frame
    // first label of each row position in this chunk (pair first members / everything else): emission prefetch
    int labp0 = -1, labp1 = -1;
    for (int q = se - 1; q >= sb; --q) { if (__ldg(P.state_pos + q)) labp1 = __ldg(P.state_label + q); else labp0 = __ldg(P.state_label + q); }
    unsigned epoch = 0;
    const int n_batches = (ae - ab) / (SMALL ? kSmallRows : BATCH);   // (small batches: kSmallRows rows per ring stage)
    const uint4 *const arc4 = SMEM_ARCS ? reinterpret_cast<const uint4 *>(s_arcs + (ab - tile_a0))
                                        : reinterpret_cast<const uint4 *>(P.arcs + ab);
    TmaRing ring{0u, 0u, 0u};
    if (SMALL) {
        ring.buf = smem_u32(smem_raw + P.ring_off) + (uint32_t)warp * kSmallRingWarpBytes;
        ring.bar = smem_u32(smem_raw + P.bar_off) + (uint32_t)warp * kSmallBarWarpBytes;
        if (lane == 0) {
            for (int st = 0; st < kSmallStages; ++st) mbar_init(ring.bar + 8u * st, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncwarp();
    }

    // per-row metadata lives in shared memory: L1 is invalidated at every grid barrier, and a global load on the
    // row-end path would cost an L2 round trip per row
    for (int i = tid; i < tile_s1 - tile_s0; i += kDenThreads) s_label[i] = __ldg(P.state_label + tile_s0 + i);
    const uint32_t row_bytes = (uint32_t)Npad * 4u;
    if (SMEM_ARCS) {   // stage the tile once, quad-wise transposed: {byte offset 0..3}{w0..3}
        uint4 *sq = reinterpret_cast<uint4 *>(s_arcs);
        const uint4 *src = reinterpret_cast<const uint4 *>(P.arcs + tile_a0);
        for (int i = tid; i < (tile_a1 - tile_a0) / kQuad; i += kDenThreads) {
            const uint4 m0 = __ldg(src + 2 * i), m1 = __ldg(src + 2 * i + 1);
            const uint32_t mul = SMALL ? 1u : row_bytes;   // TMA: row coordinates; register gathers: byte offsets
            uint4 pr = make_uint4(fwd_row(m0.x, S) * mul, fwd_row(m0.z, S) * mul, fwd_row(m1.x, S) * mul, fwd_row(m1.z, S) * mul);
            if (SMALL) {
                // zero-weight padding slots name a row coordinate beyond the tensor: the TMA unit zero-fills them in shared
                // memory without touching L2 (17 % of the forward stream; the register path gets these from L1 instead)
                if ((m0.y & 0x7fffffffu) == 0u) pr.x = kOobRow;
                if ((m0.w & 0x7fffffffu) == 0u) pr.y = kOobRow;
                if ((m1.y & 0x7fffffffu) == 0u) pr.z = kOobRow;
                if ((m1.w & 0x7fffffffu) == 0u) pr.w = kOobRow;
            }
            sq[2 * i] = pr;
            sq[2 * i + 1] = make_uint4(m0.y, m0.w, m1.y, m1.w);
        }
    }
    for (int i = tid; i < Npad; i += kDenThreads) s_sum[i] = 0.f;

    // t = 0: alpha_0 = indicator(start) (virtual rows: the pair sum); column sum 1.  Recompute of a segment: frame t_lo is
    // its checkpoint's real rows, and its pair-sum rows are rebuilt from them (the same fp32 sum the frame's row ends formed)
    {
        const bool recompute = P.ckpt_mode == 2;
        const float *src = recompute ? P.ckpt + (size_t)(P.t_lo / P.ckpt_k) * frame_elems : nullptr;
        float *a0 = P.alpha + (size_t)alpha_pos(P, P.t_lo) * frame_elems;
        auto first = [&](int q, int n) { return recompute ? __ldcg(src + (size_t)q * Npad + n) : (q == P.start ? 1.f : 0.f); };
        for (int q = sb; q < se; ++q)
            for (int n = lane; n < Npad; n += 32) __stcg(a0 + (size_t)q * Npad + n, first(q, n));
        int vj = vj0;
        for (int q = sb; q < se; ++q) {
            if (__ldg(P.state_pos + q) == 0) {   // q, q+1 are a pair
                for (int n = lane; n < Npad; n += 32) __stcg(a0 + (size_t)(virt0 + vj) * Npad + n, first(q, n) + first(q + 1, n));
                ++vj;
            }
        }
        if (cta == 0 && !recompute) for (int n = tid; n < Npad; n += kDenThreads) __stcg(P.colsum_a + n, 1.f);
    }
    // rows of high in-degree states are accumulated with atomics from several parts: zero them one frame ahead
    auto zero_hub_rows = [&](int frame) {
        float *fr = P.alpha + (size_t)alpha_pos(P, frame) * frame_elems;
        for (int i = cta * kDenThreads + tid; i < P.n_hubs * Npad; i += gridDim.x * kDenThreads)
            __stcg(fr + (size_t)__ldg(P.hub_states + i / Npad) * Npad + (i % Npad), 0.f);
    };
    if (HUBS && P.t_lo < P.t_hi) zero_hub_rows(P.t_lo + 1);
    const int my_len = (cta == 0 && tid < P.N) ? __ldg(P.len + tid) : 0;   // CTA 0 keeps log-scale books
    int len0[U];   // lengths of this lane's utterances in lane group 0 (the only group for N <= 32*U)
#pragma unroll
    for (int u = 0; u < U; ++u) len0[u] = (ul * U + u < P.N) ? __ldg(P.len + ul * U + u) : 0;
    double runlog = 0.0;
    if (SMALL) fence_proxy_async_global();
    grid_barrier(P.barrier, (++epoch) * gridDim.x);
    if (P.ckpt_mode == 1) ckpt_frame_done(P, 0, P.alpha, sb, se, lane);

    for (int t = P.t_lo + 1; t <= P.t_hi; ++t) {
        tl_mark(P, t, chunk, n_chunks, 0, lane);
        if (SMALL) fence_proxy_async_global();
        const int p_prev = alpha_pos(P, t - 1);
        const float *a_prev = P.alpha + (size_t)p_prev * frame_elems;
        float *a_cur = P.alpha + (size_t)alpha_pos(P, t) * frame_elems;
        for (int gc = 0; gc < (LPR == 32 ? Npad / (32 * U) : 1); ++gc) {
            const int n0 = gc * 32 * U + ul * U;
            bool act[U];
            bool lane_act = false;
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int ln = gc == 0 ? len0[u] : ((n0 + u < P.N) ? __ldg(P.len + n0 + u) : 0);
                act[u] = t <= ln;
                lane_act |= act[u];
            }
            if (!__any_sync(kFull, lane_act)) continue;
            float r[U], fm[U], sum[U], ypre0[U], ypre1[U], ec0[U], ec1[U];
#pragma unroll
            for (int u = 0; u < U; ++u) { r[u] = 1.f; fm[u] = 0.f; ypre0[u] = 0.f; ypre1[u] = 0.f; ec0[u] = 0.f; ec1[u] = 0.f; sum[u] = 0.f; }
            // own-row terms (den_graph.h DenPlan::own_rows): the previous frame's rows of the NEXT group to end (rows `row`,
            // `row + 1`: this warp wrote them one frame ago) and their coefficients, fetched one group ahead of use
            const bool own = P.own != 0;
            const char *const x_base = reinterpret_cast<const char *>(a_prev + n0);
            Vec<U> xa = vec_zero<U>(), xb = vec_zero<U>();
            float2 c01 = make_float2(0.f, 0.f), c23 = make_float2(0.f, 0.f);
            auto own_prefetch = [&](uint32_t row) {
                if (!own || (int)row >= se) return;
                c01 = __ldg(reinterpret_cast<const float2 *>(P.own_c) + row);
                c23 = __ldg(reinterpret_cast<const float2 *>(P.own_c) + row + 1);
                if (SMALL || lane_act) {
                    xa = gather_row<U>(x_base, row * row_bytes);
                    if ((int)row + 1 < se) xb = gather_row<U>(x_base, (row + 1u) * row_bytes);
                }
            };
            auto frame_scalars = [&]() {
                own_prefetch((uint32_t)sb);
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    int sh;
                    r[u] = scale_from_sum(__ldcg(P.colsum_a + (size_t)(t - 1) * Npad + n0 + u), &sh, P.scale_exp);
                    fm[u] = act[u] ? __ldg(P.fmax + (size_t)(t - 1) * Npad + n0 + u) : 0.f;
                    // emissions of the chunk's first labels: issued now, consumed at the first row ends
                    const long yb = (n0 + u) * P.sn + (long)(t - 1) * P.st;
                    ypre0[u] = (act[u] && labp0 >= 0) ? load_y(P.y, P.y_dtype, yb + labp0) : 0.f;
                    ypre1[u] = (act[u] && labp1 >= 0) ? load_y(P.y, P.y_dtype, yb + labp1) : 0.f;
                }
            };
            int ql = sb - tile_s0;                               // row index inside the CTA tile
            uint32_t out_row = (uint32_t)sb;                     // row q of the frame
            uint32_t virt_row = virt0 + (uint32_t)vj0;           // the next virtual row (parked two frames ahead)
            float *const out_base = a_cur + n0;
            Vec<U> cacc = vec_zero<U>();
            bool ec0_fresh = false;   // merged pairs: the first members' common emission, refreshed at the frame's first pair
            auto seg_end = [&](float *acc, int ev, bool new_label, const uint4 *quad, const float *a2, const Vec<U> &v3, float w3) {
                const bool k1 = ev != kEvRowPos0;
                if (!HUBS && ev == kEvPairMerged) {
                    // BOTH rows of a pair (den_graph.h DenPlan::fwd_merged): the second member's sum is everything but the last
                    // slot (a2), the first member's single arc is the last slot (w3 * v3); rows out_row, out_row + 1
                    if (new_label) {
                        const int lab = s_label[ql + 1];
#pragma unroll
                        for (int u = 0; u < U; ++u) {
                            const float yv = (lab == labp1) ? ypre1[u]
                                             : (act[u] ? load_y(P.y, P.y_dtype, (n0 + u) * P.sn + (long)(t - 1) * P.st + lab) : 0.f);
                            ec1[u] = act[u] ? expf(yv - fm[u]) : 0.f;
                        }
                    }
                    if (!ec0_fresh) {
#pragma unroll
                        for (int u = 0; u < U; ++u) ec0[u] = act[u] ? expf(ypre0[u] - fm[u]) : 0.f;
                        ec0_fresh = true;
                    }
                    Vec<U> o0, o1, ov;
#pragma unroll
                    for (int u = 0; u < U; ++u) {
                        // with own-row terms the segment has no tail slot: both rows take their own-group part from xa / xb
                        const float s0 = own ? fmaf(c01.x, xa.v[u], c01.y * xb.v[u]) : w3 * v3.v[u];
                        const float s1 = own ? fmaf(c23.x, xa.v[u], fmaf(c23.y, xb.v[u], acc[u])) : a2[u];
                        o0.v[u] = s0 * ec0[u] * r[u];   // (no own terms: same operation order as a one-arc row, fma(w, v, 0) * e * r)
                        o1.v[u] = s1 * ec1[u] * r[u];
                        if (SMALL && !act[u]) { o0.v[u] = 0.f; o1.v[u] = 0.f; }
                        ov.v[u] = o0.v[u] + o1.v[u];
                        sum[u] += o0.v[u];
                        sum[u] += o1.v[u];
                        acc[u] = 0.f;
                    }
                    if ((SMALL || lane_act) && sub == 0) {
                        o0.stcg(row_ptr<U>(out_base, out_row, row_bytes));
                        o1.stcg(row_ptr<U>(out_base, out_row + 1u, row_bytes));
                        ov.stcg(row_ptr<U>(out_base, virt_row, row_bytes));
                    }
                    ++virt_row;
                    out_row += 2u;
                    ql += 2;
                    own_prefetch(out_row);
                    return;
                }
                if (HUBS && ev == kEvPartial) {   // high in-degree rows only: handled out of line, nothing hot is captured
                    Vec<U> part;
#pragma unroll
                    for (int u = 0; u < U; ++u) { part.v[u] = acc[u]; acc[u] = 0.f; }
                    // byte offset of the target row (last slot of the segment)
                    const uint32_t tgt_off = load_quad_peers<SMEM_ARCS>(quad, row_bytes, (uint32_t)S).w;
                    forward_partial_row<U>(P.state_label, P.len, P.colsum_a + (size_t)(t - 1) * Npad, P.fmax + (size_t)(t - 1) * Npad,
                                           P.y, P.y_dtype, P.sn, (long)(t - 1) * P.st, P.N, t, n0, part, tgt_off, row_bytes, a_cur, s_sum, P.scale_exp);
                    if (tgt_off == out_row * row_bytes) { ++out_row; ++ql; }   // the part that lives in the row's own group
                    return;
                }
                if (new_label) {   // rare: a new label for this row position -> refresh its emission
                    const int lab = s_label[ql];
                    const int lp = k1 ? labp1 : labp0;
#pragma unroll
                    for (int u = 0; u < U; ++u) {
                        const float yv = (lab == lp) ? (k1 ? ypre1[u] : ypre0[u])
                                         : (act[u] ? load_y(P.y, P.y_dtype, (n0 + u) * P.sn + (long)(t - 1) * P.st + lab) : 0.f);
                        const float en = act[u] ? expf(yv - fm[u]) : 0.f;
                        if (k1) ec1[u] = en; else ec0[u] = en;
                    }
                }
                Vec<U> out;
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    if (own) acc[u] = fmaf(c01.y, xa.v[u], acc[u]);     // unpaired row: its own previous-frame value (self loop)
                    out.v[u] = acc[u] * (k1 ? ec1[u] : ec0[u]) * r[u];   // ec is 0 for inactive utterances
                    // TMA rows are read by every lane, whatever its utterances do: inactive columns are kept at a clean 0
                    // (the register path never loads them)
                    if (SMALL && !act[u]) out.v[u] = 0.f;
                    sum[u] += out.v[u];
                    acc[u] = 0.f;
                }
                if ((SMALL || lane_act) && sub == 0) out.stcg(row_ptr<U>(out_base, out_row, row_bytes));
                if (ev == kEvRowPos0) cacc = out;
                else if (ev == kEvRowPos1) {   // the pair's virtual row: what the next frame gathers instead of both
#pragma unroll
                    for (int u = 0; u < U; ++u) cacc.v[u] += out.v[u];
                    if ((SMALL || lane_act) && sub == 0) cacc.stcg(row_ptr<U>(out_base, virt_row, row_bytes));
                    ++virt_row;
                }
                ++out_row;
                ++ql;
                own_prefetch(out_row);
            };
            if (SMALL) {
                float acc[1] = {0.f};
                walk_arcs_tma_small<2>(arc4, n_batches, P.alpha, p_prev * S, ring, lane, frame_scalars,
                                       [&](const uint4 *quad, const float *v, uint32_t) {
                    const uint4 wq = quad[1];
                    float before = acc[0];   // the lane's sum before the quad's last LDS step (slot 3 = last step of lane group 1)
#pragma unroll
                    for (int st = 0; st < 2; ++st) {
                        if (st == 1) before = acc[0];
                        acc[0] = fmaf(fabsf(__uint_as_float(quad_word(wq, st * 2 + sub))), v[st], acc[0]);
                    }
                    if ((int)wq.w < 0) {   // warp-uniform: a segment ends at this quad -> combine the lane groups' partial sums
                        const int ev = (int)(((wq.z >> 31) << 1) | (wq.y >> 31));
                        float a2[1] = {0.f};
                        Vec<U> v3 = vec_zero<U>();   // (U == 1 on this path)
                        if (ev == kEvPairMerged && !own) {   // slot 3 (the pair's first member) apart from the rest (its second member)
                            const bool last = sub == 1;
                            a2[0] = last ? before : acc[0];
                            v3.v[0] = last ? fabsf(__uint_as_float(wq.w)) * v[1] : 0.f;
                            a2[0] += __shfl_xor_sync(kFull, a2[0], 16);
                            v3.v[0] += __shfl_xor_sync(kFull, v3.v[0], 16);
                        } else {
                            acc[0] += __shfl_xor_sync(kFull, acc[0], 16);
                        }
                        seg_end(acc, ev, (int)wq.x < 0, quad, a2, v3, 1.f);
                    }
                });
            } else {
                walk_arcs<U, BATCH, SMEM_ARCS>(arc4, n_batches, row_bytes, (uint32_t)S, reinterpret_cast<const char *>(a_prev + n0), lane_act,
                                               frame_scalars, seg_end);
            }
#pragma unroll
            for (int u = 0; u < U; ++u)
                if (act[u] && sub == 0 && sum[u] != 0.f) atomicAdd(&s_sum[n0 + u], sum[u]);
        }
        tl_mark(P, t, chunk, n_chunks, 1, lane);
        if (HUBS && t < P.t_hi) zero_hub_rows(t + 1);
        if (SMALL) fence_proxy_async_global();   // this frame's rows are read through the async proxy after the barrier
        __syncthreads();
        for (int i = tid; i < Npad; i += kDenThreads) {   // (a recompute reads the first pass's column sums, it does not add to them)
            const float v = s_sum[i];
            if (v != 0.f) { if (P.ckpt_mode != 2) atomicAdd(P.colsum_a + (size_t)t * Npad + i, v); s_sum[i] = 0.f; }
        }
        // arrive first, then the log-scale books of CTA 0 (two L2 round trips nobody waits for) in the barrier's shadow
        grid_barrier_arrive(P.barrier);
        if (cta == 0 && tid < P.N && t <= my_len) {
            int sh;
            (void)scale_from_sum(__ldcg(P.colsum_a + (size_t)(t - 1) * Npad + tid), &sh, P.scale_exp);
            runlog += (double)__ldg(P.fmax + (size_t)(t - 1) * Npad + tid) - (double)sh * 0.6931471805599453;
        }
        grid_barrier_wait(P.barrier, (++epoch) * gridDim.x);
        tl_mark(P, t, chunk, n_chunks, 2, lane);
        // (frame t's position is rewritten kAlphaRing frames later)
        if (P.ckpt_mode == 1) ckpt_frame_done(P, t, P.alpha + (size_t)alpha_pos(P, t) * frame_elems, sb, se, lane);
    }
    if (P.ckpt_mode == 2) return;   // a recompute only refills the segment's frames

    // logZ[n] = log sum_q alpha_len(q) final(q) + accumulated log scale      (den_calculate.cu:105-161)
    // (first checkpointed pass: already summed into zsum frame by frame, ckpt_frame_done)
    for (int gc = 0; gc < (P.ckpt_mode == 0 ? (Npad + 31) / 32 : 0); ++gc) {
        const int n = gc * 32 + lane;
        const int ln = (n < P.N) ? __ldg(P.len + n) : -1;
        float zs = 0.f;
        if (ln >= 0) {
            for (int q = sb; q < se; ++q) {
                const float f = __ldg(P.final_lin + q);
                if (f != 0.f) zs = fmaf(f, __ldcg(P.alpha + (size_t)ln * frame_elems + (size_t)q * Npad + n), zs);
            }
        }
        if (zs != 0.f) atomicAdd(&s_sum[n], zs);
    }
    __syncthreads();
    for (int i = tid; i < Npad; i += kDenThreads) {
        const float v = s_sum[i];
        if (v != 0.f) atomicAdd(P.zsum + i, v);
    }
    grid_barrier(P.barrier, (++epoch) * gridDim.x);
    if (cta == 0 && tid < P.N) P.logz[tid] = (float)(log((double)__ldcg(P.zsum + tid)) + runlog - (P.lnorm ? P.lnorm[tid] : 0.0));
}

// ------------------------------------------------------------------------------------------------
// backward: beta recursion, occupancies, logZ from beta
// ------------------------------------------------------------------------------------------------
// Rows are gathered into registers (walk_arcs_dual) except in two TMA variants: SMALL, the small-batch variant
// (walk_arcs_tma_small, 16 lanes per row, arc tile in shared memory, one utterance per lane), and STREAM, the streamed-arc
// tier (walk_arcs_tma_stream, full-width rows, arcs flowing through per-warp rings).
template <int U, int BATCH, bool SMEM_ARCS, bool W1_SMEM = SMEM_ARCS, bool SMALL = false, bool STREAM = false>
__global__ void __launch_bounds__(kDenThreads, 1) den_backward_kernel(const __grid_constant__ DenParams P) {
    constexpr bool TMA = SMALL || STREAM;
    constexpr int LPR = SMALL ? kSmallLanes : 32;   // lanes per row
    static_assert(!SMALL || (SMEM_ARCS && U == 1), "small-batch variant: arc tile in shared memory, one utterance per lane");
    static_assert(!STREAM || (!SMEM_ARCS && !SMALL), "streamed arcs: not resident, full-width rows");
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int Npad = P.Npad, S = P.S;
    float *s_sum = reinterpret_cast<float *>(smem_raw);            // [2][Npad]: colsum_b, absum
    float *s_gacc = s_sum + 2 * Npad;                              // [gacc_rows][Npad]
    int *s_label = reinterpret_cast<int *>(s_gacc + (size_t)P.gacc_rows * Npad);   // [tile_rows]
    float *s_final = reinterpret_cast<float *>(s_label + P.tile_rows);             // [tile_rows]
    Arc *s_arcs = reinterpret_cast<Arc *>(smem_raw + BwdArcsOff(Npad, P.gacc_rows, P.tile_rows));

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(kFull, tid >> 5, 0);   // (through a shuffle: lets ptxas keep warp-derived addresses in uniform registers)
    const int sub = LPR == 32 ? 0 : lane / LPR;    // small batches: which arc(s) of a quad this lane multiplies
    const int ul = LPR == 32 ? lane : lane % LPR;   // ... and which utterance it carries (lane groups sub > 0 are replicas at row ends)
    const int cta = blockIdx.x;
    const int chunk = cta * P.n_warps + warp;
    const int n_chunks = gridDim.x * P.n_warps;
    const int sb = __ldg(P.chunk_state + chunk), se = __ldg(P.chunk_state + chunk + 1);
    const int ab = __ldg(P.chunk_arc + chunk), ae = __ldg(P.chunk_arc + chunk + 1);
    const int tile_a0 = __ldg(P.chunk_arc + cta * P.n_warps);
    const int tile_a1 = __ldg(P.chunk_arc + (cta + 1) * P.n_warps);
    const int tile_s0 = __ldg(P.chunk_state + cta * P.n_warps);
    const int tile_s1 = __ldg(P.chunk_state + (cta + 1) * P.n_warps);
    // label accumulator rows of this CTA: [cl_n0 labels from cl_lab0 (pair first members)] [cl_n1 from cl_lab1 (others)]
    const int cl_lab0 = __ldg(P.cta_labels + cta * 4), cl_n0 = __ldg(P.cta_labels + cta * 4 + 1);
    const int cl_lab1 = __ldg(P.cta_labels + cta * 4 + 2), cl_n1 = __ldg(P.cta_labels + cta * 4 + 3);
    int labp0 = -1, labp1 = -1;
    for (int q = se - 1; q >= sb; --q) { if (__ldg(P.state_pos + q)) labp1 = __ldg(P.state_label + q); else labp0 = __ldg(P.state_label + q); }
    const int n_batches = (ae - ab) / (SMALL ? kSmallRows : BATCH);   // (small batches: kSmallRows rows per ring stage; streamed arcs: BATCH)
    // shared memory: 3 words of 16 bytes per quad {byte offsets}{w0}{w1}; global fallback: AoS arcs + w1 array
    constexpr int kW = W1_SMEM ? 3 : 2;   // 16-byte words per staged quad
    const uint4 *const arc4 = SMEM_ARCS ? reinterpret_cast<const uint4 *>(s_arcs) + kW * ((ab - tile_a0) / kQuad)
                                        : reinterpret_cast<const uint4 *>(P.arcs + ab);
    const float4 *const w1g = reinterpret_cast<const float4 *>(P.w1 + ab);
    const bool use_gacc = P.gacc_rows > 0;
    const size_t frame_elems = (size_t)S * Npad;                         // beta ping-pong: real rows only
    const size_t alpha_frame = (size_t)S * Npad;                          // alpha spill: real rows only (see den_forward_kernel)
    unsigned epoch = 0;

    for (int i = tid; i < tile_s1 - tile_s0; i += kDenThreads) {
        s_label[i] = __ldg(P.state_label + tile_s0 + i);
        s_final[i] = __ldg(P.final_lin + tile_s0 + i);
    }
    const uint32_t row_bytes = (uint32_t)Npad * 4u;
    if (SMEM_ARCS) {   // stage the tile once, quad-wise transposed: {byte offset 0..3}{w0 0..3}[{w1 0..3}]
        uint4 *sq = reinterpret_cast<uint4 *>(s_arcs);
        const uint4 *src = reinterpret_cast<const uint4 *>(P.arcs + tile_a0);
        const uint4 *src1 = reinterpret_cast<const uint4 *>(P.w1 + tile_a0);
        for (int i = tid; i < (tile_a1 - tile_a0) / kQuad; i += kDenThreads) {
            const uint4 m0 = __ldg(src + 2 * i), m1 = __ldg(src + 2 * i + 1);
            const uint32_t mul = TMA ? 1u : row_bytes;   // TMA: row coordinates; register gathers: byte offsets
            uint4 pr = make_uint4(m0.x * mul, m0.z * mul, m1.x * mul, m1.z * mul);
            const uint4 w1q = __ldg(src1 + i);
            if (TMA) {   // padding slots (both weights zero): out-of-bounds row coordinate, zero-filled by the TMA unit
                if ((m0.y & 0x7fffffffu) == 0u && w1q.x == 0u) pr.x = kOobRow;
                if ((m0.w & 0x7fffffffu) == 0u && w1q.y == 0u) pr.y = kOobRow;
                if ((m1.y & 0x7fffffffu) == 0u && w1q.z == 0u) pr.z = kOobRow;
                if ((m1.w & 0x7fffffffu) == 0u && w1q.w == 0u) pr.w = kOobRow;
            }
            sq[kW * i] = pr;
            sq[kW * i + 1] = make_uint4(m0.y, m0.w, m1.y, m1.w);
            if (W1_SMEM) sq[kW * i + 2] = w1q;
        }
    }
    TmaRing ring{0u, 0u, 0u};
    if (TMA) {
        constexpr int kStages = SMALL ? kSmallStages : 2;
        ring.buf = smem_u32(smem_raw + P.ring_off) + (uint32_t)warp * (SMALL ? kSmallRingWarpBytes : StreamRingWarpBytes(U));
        ring.bar = smem_u32(smem_raw + P.bar_off) + (uint32_t)warp * (SMALL ? kSmallBarWarpBytes : kStreamBarWarpBytes);
        if (lane == 0) {
            for (int st = 0; st < kStages; ++st) mbar_init(ring.bar + 8u * st, 1);
            if (STREAM) for (int st = 0; st < kArcStages; ++st) mbar_init(smem_u32(smem_raw + P.abar_off) + (uint32_t)(warp * (kArcBarWarpBytes / 8) + st) * 8u, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncwarp();
    }
    ArcRing aring{nullptr, 0u, 0u, 0u, 0u, 0u, 0u, nullptr};
    if (STREAM) {
        constexpr int kAW = BATCH / kQuad * 3;   // 16-byte words per batch
        aring.buf = reinterpret_cast<const uint4 *>(smem_raw + P.aring_off) + (size_t)warp * (kArcRingWarpBytes / 16);
        aring.buf_s = smem_u32(aring.buf);
        aring.bar = smem_u32(smem_raw + P.abar_off) + (uint32_t)warp * kArcBarWarpBytes;
        aring.n = (uint32_t)n_batches;
        aring.src = P.tq + (size_t)3 * (ab / kQuad);
        arc_ring_fill<kAW>(aring, lane);
    }
    for (int i = tid; i < (2 + P.gacc_rows) * Npad; i += kDenThreads) s_sum[i] = 0.f;
    const int my_len = (cta == 0 && tid < P.N) ? __ldg(P.len + tid) : 0;
    int len0[U];
#pragma unroll
    for (int u = 0; u < U; ++u) len0[u] = (ul * U + u < P.N) ? __ldg(P.len + ul * U + u) : 0;
    double runlog = 0.0;
    // segmented backward pass (checkpointed alpha): beta-hat, colsum_b and absum carry over in global memory, the
    // log-scale books through runlog_b
    if (P.t_hi < P.Tmax && cta == 0 && tid < P.N) runlog = P.runlog_b[tid];
    __syncthreads();

    for (int tau = P.t_hi; tau > P.t_lo; --tau) {
        tl_mark(P, P.Tmax - tau, chunk, n_chunks, 0, lane);
        if (TMA) fence_proxy_async_global();
        const float *bh_next = P.bh + (size_t)((tau + 1) & 1) * frame_elems;
        float *bh_cur = P.bh + (size_t)(tau & 1) * frame_elems;
        // alpha_pos without the ring (a_ring = 0 for every backward launch): frame tau - 1 is the position before frame tau
        const float *a_row = P.alpha + (size_t)(tau - P.a_base) * alpha_frame;
        if (tau > 1 && se > sb) {   // pull next step's alpha rows of this chunk towards L2
            const char *nb = reinterpret_cast<const char *>(a_row - alpha_frame + (size_t)sb * Npad);
            const size_t bytes = (size_t)(se - sb) * Npad * 4;
            for (size_t off = (size_t)lane * 128; off < bytes; off += 32 * 128) prefetch_l2(nb + off);
        }
        for (int gc = 0; gc < (LPR == 32 ? Npad / (32 * U) : 1); ++gc) {
            const int n0 = gc * 32 * U + ul * U;
            bool act[U], gat[U];
            bool lane_act = false, lane_gat = false;
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int ln = gc == 0 ? len0[u] : ((n0 + u < P.N) ? __ldg(P.len + n0 + u) : 0);
                act[u] = tau <= ln;      // beta_tau exists
                gat[u] = tau < ln;       // ... and is a sum over arcs (tau == len: final weights)
                lane_act |= act[u];
                lane_gat |= gat[u];
            }
            if (!__any_sync(kFull, lane_act)) continue;
            float rb[U], fm[U], sum_b[U], sum_ab[U], gsum0[U], gsum1[U], ypre0[U], ypre1[U], ec0[U], ec1[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                rb[u] = 1.f; fm[u] = 0.f; ypre0[u] = 0.f; ypre1[u] = 0.f; ec0[u] = 0.f; ec1[u] = 0.f;
                gsum0[u] = 0.f; gsum1[u] = 0.f; sum_b[u] = 0.f; sum_ab[u] = 0.f;
            }
            auto frame_scalars = [&]() {
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    int sh;
                    rb[u] = gat[u] ? scale_from_sum(__ldcg(P.colsum_b + (size_t)(tau + 1) * Npad + n0 + u), &sh, P.scale_exp) : 1.f;
                    fm[u] = act[u] ? __ldg(P.fmax + (size_t)(tau - 1) * Npad + n0 + u) : 0.f;
                    const long yb = (n0 + u) * P.sn + (long)(tau - 1) * P.st;
                    ypre0[u] = (act[u] && labp0 >= 0) ? load_y(P.y, P.y_dtype, yb + labp0) : 0.f;
                    ypre1[u] = (act[u] && labp1 >= 0) ? load_y(P.y, P.y_dtype, yb + labp1) : 0.f;
                }
            };
            int curlab0 = -1, curlab1 = -1;
            int ql = sb - tile_s0;
            uint32_t out_row = (uint32_t)sb;
            float *const out_base = bh_cur + n0;
            const char *const a_base = reinterpret_cast<const char *>(a_row + n0);
            // alpha rows of the next group (one or two states) are fetched one group ahead
            Vec<U> a_q = (se > sb && lane_act) ? gather_row<U>(a_base, out_row * row_bytes) : vec_zero<U>();
            Vec<U> a_q1 = (se > sb + 1 && lane_act) ? gather_row<U>(a_base, (out_row + 1) * row_bytes) : vec_zero<U>();
            // own-row terms (den_graph.h DenPlan::own_rows): the next frame's beta-hat rows of the group about to end (this warp
            // wrote them one frame ago) and their coefficients, fetched one group ahead like the alpha rows
            const bool own = P.own != 0;
            const char *const b_base = reinterpret_cast<const char *>(bh_next + n0);
            Vec<U> xa = vec_zero<U>(), xb = vec_zero<U>();
            float2 c01 = make_float2(0.f, 0.f), c23 = make_float2(0.f, 0.f);
            auto own_prefetch = [&](uint32_t row) {
                if (!own || (int)row >= se) return;
                c01 = __ldg(reinterpret_cast<const float2 *>(P.own_c) + row);
                c23 = __ldg(reinterpret_cast<const float2 *>(P.own_c) + row + 1);
                if (TMA || lane_act) {
                    xa = gather_row<U>(b_base, row * row_bytes);
                    if ((int)row + 1 < se) xb = gather_row<U>(b_base, (row + 1u) * row_bytes);
                }
            };
            own_prefetch(out_row);
            auto flush_gsum = [&](bool k1) {
                const int lab = k1 ? curlab1 : curlab0;
                const int row = k1 ? cl_n0 + lab - cl_lab1 : lab - cl_lab0;
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const float g = k1 ? gsum1[u] : gsum0[u];
                    if (g != 0.f && sub == 0) {
                        if (use_gacc) atomicAdd(&s_gacc[row * Npad + n0 + u], g);
                        else atomicAdd(P.grad + (n0 + u) * P.gsn + (long)(tau - 1) * P.gst + lab, g);
                    }
                    if (k1) gsum1[u] = 0.f; else gsum0[u] = 0.f;
                }
            };
            // one state's row end: beta_tau(q), its occupancy, the emission-weighted value the next frame gathers
            auto do_row = [&](bool k1, bool new_label, float *acc, const Vec<U> &a_val) {
                if (new_label) {
                    const int lab = s_label[ql];
                    if ((k1 ? curlab1 : curlab0) >= 0) flush_gsum(k1);
                    const int lp = k1 ? labp1 : labp0;
#pragma unroll
                    for (int u = 0; u < U; ++u) {
                        const float yv = (lab == lp) ? (k1 ? ypre1[u] : ypre0[u])
                                         : (act[u] ? load_y(P.y, P.y_dtype, (n0 + u) * P.sn + (long)(tau - 1) * P.st + lab) : 0.f);
                        const float en = act[u] ? expf(yv - fm[u]) : 0.f;
                        if (k1) ec1[u] = en; else ec0[u] = en;
                    }
                    if (k1) curlab1 = lab; else curlab0 = lab;
                }
                const float f = s_final[ql];
                Vec<U> out;
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const float b = act[u] ? (gat[u] ? acc[u] * rb[u] : f) : 0.f;
                    const float abp = a_val.v[u] * b;          // a_val is 0 for inactive lanes
                    if (k1) gsum1[u] += abp; else gsum0[u] += abp;
                    sum_ab[u] += abp;
                    out.v[u] = (k1 ? ec1[u] : ec0[u]) * b;
                    sum_b[u] += out.v[u];
                    acc[u] = 0.f;
                }
                if ((TMA || lane_act) && sub == 0) out.stcg(row_ptr<U>(out_base, out_row, row_bytes));   // (TMA: every lane reads the row later)
                ++out_row;
                ++ql;
            };
            auto group_end = [&](float *acc0, float *acc1, bool pair, bool new0, bool new1) {
                if (own) {
#pragma unroll
                    for (int u = 0; u < U; ++u) {
                        if (pair) {
                            acc0[u] = fmaf(c01.x, xa.v[u], fmaf(c01.y, xb.v[u], acc0[u]));
                            acc1[u] = fmaf(c23.x, xa.v[u], fmaf(c23.y, xb.v[u], acc1[u]));
                        } else {
                            acc0[u] = fmaf(c01.y, xa.v[u], acc0[u]);   // unpaired row: its own next-frame value (self loop)
                        }
                    }
                }
                if (pair) {
                    do_row(false, new0, acc0, a_q);
                    do_row(true, new1, acc1, a_q1);
                } else {
                    do_row(true, new0, acc0, a_q);
#pragma unroll
                    for (int u = 0; u < U; ++u) acc1[u] = 0.f;
                }
                a_q = ((int)out_row < se && lane_act) ? gather_row<U>(a_base, out_row * row_bytes) : vec_zero<U>();
                a_q1 = ((int)out_row + 1 < se && lane_act) ? gather_row<U>(a_base, (out_row + 1) * row_bytes) : vec_zero<U>();
                own_prefetch(out_row);
            };
            if (SMALL) {
                float acc0[1] = {0.f}, acc1[1] = {0.f};
                const uint32_t w1buf = SmallW1Off(smem_u32(smem_raw + P.bar_off), P.n_warps) + (uint32_t)warp * kSmallW1WarpBytes;
                walk_arcs_tma_small<W1_SMEM ? 3 : 2, !W1_SMEM>(arc4, n_batches, P.bh, ((tau + 1) & 1) * S, ring, lane, frame_scalars,
                                                               [&](const uint4 *quad, const float *v, uint32_t w1s) {
                    const uint4 wq = quad[1];
                    uint4 t1;
                    if (W1_SMEM) t1 = quad[2];
                    else asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(t1.x), "=r"(t1.y), "=r"(t1.z), "=r"(t1.w) : "r"(w1s));
#pragma unroll
                    for (int st = 0; st < 2; ++st) {
                        const int j = st * 2 + sub;
                        acc0[0] = fmaf(fabsf(__uint_as_float(quad_word(wq, j))), v[st], acc0[0]);
                        acc1[0] = fmaf(__uint_as_float(quad_word(t1, j)), v[st], acc1[0]);
                    }
                    if ((int)wq.w < 0) {   // warp-uniform: the group ends at this quad -> combine the lane groups' partial sums
                        acc0[0] += __shfl_xor_sync(kFull, acc0[0], 16);
                        acc1[0] += __shfl_xor_sync(kFull, acc1[0], 16);
                        group_end(acc0, acc1, (int)wq.z < 0, (int)wq.x < 0, (int)wq.y < 0);
                    }
                }, reinterpret_cast<const float *>(w1g), w1buf);
            } else if (STREAM) {
                float acc0[U], acc1[U];
#pragma unroll
                for (int u = 0; u < U; ++u) { acc0[u] = 0.f; acc1[u] = 0.f; }
                // (the first backward frame of an utterance takes beta from the final weights, not from these sums: whatever
                // the ring holds then is never selected, see do_row)
                auto consume_quad = [&](const uint4 *quad, const Vec<U> *v) {
                    const uint4 wq = quad[1], t1 = quad[2];
                    const float a0 = fabsf(__uint_as_float(wq.x)), a1 = fabsf(__uint_as_float(wq.y));
                    const float a2 = fabsf(__uint_as_float(wq.z)), a3 = fabsf(__uint_as_float(wq.w));
                    const float b0 = __uint_as_float(t1.x), b1 = __uint_as_float(t1.y), b2 = __uint_as_float(t1.z), b3 = __uint_as_float(t1.w);
#pragma unroll
                    for (int u = 0; u < U; ++u) {
                        acc0[u] = fmaf(a0, v[0].v[u], acc0[u]); acc1[u] = fmaf(b0, v[0].v[u], acc1[u]);
                        acc0[u] = fmaf(a1, v[1].v[u], acc0[u]); acc1[u] = fmaf(b1, v[1].v[u], acc1[u]);
                        acc0[u] = fmaf(a2, v[2].v[u], acc0[u]); acc1[u] = fmaf(b2, v[2].v[u], acc1[u]);
                        acc0[u] = fmaf(a3, v[3].v[u], acc0[u]); acc1[u] = fmaf(b3, v[3].v[u], acc1[u]);
                    }
                    if ((int)wq.w < 0)   // warp-uniform: the group ends at this quad
                        group_end(acc0, acc1, (int)wq.z < 0, (int)wq.x < 0, (int)wq.y < 0);
                };
                walk_arcs_tma_stream<U, BATCH, 3>(aring, n_batches, &P.tmap, gc * 32 * U, ((tau + 1) & 1) * S, ring, lane, frame_scalars, consume_quad);
            } else {
                walk_arcs_dual<U, BATCH, SMEM_ARCS, W1_SMEM>(arc4, w1g, n_batches, row_bytes, reinterpret_cast<const char *>(bh_next + n0),
                                                             lane_gat, frame_scalars, group_end);
            }
            if (curlab0 >= 0) flush_gsum(false);
            if (curlab1 >= 0) flush_gsum(true);
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (act[u] && sub == 0) {
                    if (sum_b[u] != 0.f) atomicAdd(&s_sum[n0 + u], sum_b[u]);
                    if (sum_ab[u] != 0.f) atomicAdd(&s_sum[Npad + n0 + u], sum_ab[u]);
                }
            }
        }
        tl_mark(P, P.Tmax - tau, chunk, n_chunks, 1, lane);
        if (TMA) fence_proxy_async_global();   // this frame's rows are read through the async proxy after the barrier
        __syncthreads();
        for (int i = tid; i < Npad; i += kDenThreads) {   // the next frame's scale: must be out before this CTA arrives
            const float vb = s_sum[i];
            if (vb != 0.f) { atomicAdd(P.colsum_b + (size_t)tau * Npad + i, vb); s_sum[i] = 0.f; }
        }
        // Everything the next frame reads is written: arrive now, and flush what only the end of the kernel needs
        // (occupancy sums, the label accumulator) in the shadow of the barrier latency.
        grid_barrier_arrive(P.barrier);
        for (int i = tid; i < Npad; i += kDenThreads) {
            const float vab = s_sum[Npad + i];
            if (vab != 0.f) { atomicAdd(P.absum + (size_t)tau * Npad + i, vab); s_sum[Npad + i] = 0.f; }
        }
        if (use_gacc) {
            for (int i = tid; i < (cl_n0 + cl_n1) * Npad; i += kDenThreads) {
                const float g = s_gacc[i];
                if (g != 0.f) {
                    const int n = i % Npad, row = i / Npad;
                    const int k = row < cl_n0 ? cl_lab0 + row : cl_lab1 + row - cl_n0;
                    atomicAdd(P.grad + n * P.gsn + (long)(tau - 1) * P.gst + k, g);
                    s_gacc[i] = 0.f;
                }
            }
        }
        // log-scale of beta: LB_tau = LB_{tau+1} + m_tau - log rb_{tau+1}   (applies for tau < len)
        if (cta == 0 && tid < P.N && tau < my_len) {
            int sh;
            (void)scale_from_sum(__ldcg(P.colsum_b + (size_t)(tau + 1) * Npad + tid), &sh, P.scale_exp);
            runlog += (double)__ldg(P.fmax + (size_t)tau * Npad + tid) - (double)sh * 0.6931471805599453;
        }
        grid_barrier_wait(P.barrier, (++epoch) * gridDim.x);
        tl_mark(P, P.Tmax - tau, chunk, n_chunks, 2, lane);
    }

    if (STREAM) arc_ring_drain(aring);
    if (P.t_lo > 0) {   // a later segment launch continues from here
        if (cta == 0 && tid < P.N) P.runlog_b[tid] = runlog;
        return;
    }
    // tau = 0: beta_0(start) only -> logZ recomputed from the backward pass (den_calculate.cu:177-187,255-261)
    if (cta == 0 && warp == 0) {
        const float *bh1 = P.bh + (size_t)(1 & 1) * frame_elems;
        for (int n = lane; n < P.N; n += 32) {
            const int ln = __ldg(P.len + n);
            float b = P.start_final;
            if (ln > 0) {
                int sh;
                const float rb = scale_from_sum(__ldcg(P.colsum_b + (size_t)1 * Npad + n), &sh, P.scale_exp);
                float acc = 0.f;
                for (int a = 0; a < P.n_start_arcs; ++a) {
                    const Arc k = P.start_arcs[a];
                    acc = fmaf(k.w, __ldcg(bh1 + (size_t)k.peer * Npad + n), acc);
                }
                b = acc * rb;
            }
            __stcg(P.b0 + n, b);
        }
    }
    if (cta == 0 && tid < P.N && 0 < my_len) {
        int sh;
        (void)scale_from_sum(__ldcg(P.colsum_b + (size_t)1 * Npad + tid), &sh, P.scale_exp);
        runlog += (double)__ldg(P.fmax + tid) - (double)sh * 0.6931471805599453;
    }
    grid_barrier(P.barrier, (++epoch) * gridDim.x);
    if (cta == 0 && tid < P.N) P.logz[tid] = (float)(log((double)__ldcg(P.b0 + tid)) + runlog - (P.lnorm ? P.lnorm[tid] : 0.0));
}

// grad[n][t][:] *= scale / absum[t+1][n]   for t < len[n]
__global__ void den_grad_normalize_kernel(float *grad, long gsn, long gst, const float *absum, const int *len,
                                          int N, int Npad, int T, int V, float scale) {
    const long row = blockIdx.x;   // (n, t)
    const int n = (int)(row / T), t = (int)(row % T);
    if (t >= len[n]) return;
    const float s = absum[(size_t)(t + 1) * Npad + n];
    const float f = s > 0.f ? scale / s : 0.f;
    float *g = grad + n * gsn + t * gst;
    for (int k = threadIdx.x; k < V; k += blockDim.x) g[k] *= f;
}

// ------------------------------------------------------------------------------------------------
// launch plumbing
// ------------------------------------------------------------------------------------------------
int LaunchCoop(const void *fn, const DenParams &p, int n_ctas, size_t smem, cudaStream_t stream, std::string *err) {
    cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { *err = std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(e); return (int)e; }
    int per_sm = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kDenThreads, smem);
    if (e != cudaSuccess || per_sm < 1) {
        *err = "den kernel does not fit on an SM (smem=" + std::to_string(smem) + ")";
        return e != cudaSuccess ? (int)e : 1;
    }
    DenParams pc = p;
    void *args[] = {&pc};
    e = cudaLaunchCooperativeKernel(fn, dim3(n_ctas), dim3(kDenThreads), args, smem, stream);
    if (e != cudaSuccess) { *err = std::string("cooperative launch failed: ") + cudaGetErrorString(e); return (int)e; }
    CountLaunch();
    return 0;
}

// 2-D view [rows][Npad] fp32 of `base` with a box of 1 row x box_cols columns, by cuTensorMapEncodeTiled through the
// runtime's driver entry point (no link-time dependency on libcuda); false if that is unavailable or refuses the shape
bool EncodeRowTensorMap(CUtensorMap *tm, const float *base, size_t rows, int Npad, int box_cols) {
    typedef CUresult (*EncodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                    const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static EncodeTiled encode = []() -> EncodeTiled {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
            cudaGetLastError();
            return nullptr;
        }
        return (EncodeTiled)fn;
    }();
    if (!encode || !base || rows == 0 || box_cols > 256 || (reinterpret_cast<uintptr_t>(base) & 15)) return false;
    cuuint64_t dims[2] = {(cuuint64_t)Npad, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)Npad * 4};
    cuuint32_t box[2] = {(cuuint32_t)box_cols, 1};
    cuuint32_t estr[2] = {1, 1};
    return encode(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float *>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// the kernel instantiation a launch names (den_launch.h DenLaunch)
template <int U>
const void *ForwardKernel(const DenLaunch &L, bool hubs) {
    constexpr int B = FwdBatch(U);
    if (L.tier == kTierShared) return hubs ? (const void *)den_forward_kernel<U, B, true, true> : (const void *)den_forward_kernel<U, B, true, false>;
    return hubs ? (const void *)den_forward_kernel<U, B, false, true> : (const void *)den_forward_kernel<U, B, false, false>;
}
template <int U>
const void *BackwardKernel(const DenLaunch &L) {
    if (L.tier == kTierStreamed) return (const void *)den_backward_kernel<U, kStreamRows, false, true, false, true>;
    if (L.tier == kTierGlobal) return (const void *)den_backward_kernel<U, kBwdBatch, false>;
    return L.w1_smem ? (const void *)den_backward_kernel<U, kBwdBatch, true, true> : (const void *)den_backward_kernel<U, kBwdBatch, true, false>;
}
const void *DenKernel(bool backward, const DenLaunch &L, bool hubs) {
    if (L.tier == kTierSmall)
        return !backward ? (const void *)den_forward_kernel<1, kSmallRows, true, false, true>
             : L.w1_smem ? (const void *)den_backward_kernel<1, kSmallRows, true, true, true>
                         : (const void *)den_backward_kernel<1, kSmallRows, true, false, true>;
    if (backward) return L.U == 1 ? BackwardKernel<1>(L) : BackwardKernel<2>(L);
    return L.U == 1 ? ForwardKernel<1>(L, hubs) : L.U == 2 ? ForwardKernel<2>(L, hubs) : ForwardKernel<4>(L, hubs);
}

}  // namespace

DenAuxLayout MakeDenAuxLayout(int S, int N, int T, bool small_ok) {
    DenAuxLayout L;
    L.Npad = PadLanes(N, small_ok);
    auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
    size_t off = 0;
    const size_t rows = (size_t)(T + 2) * L.Npad * 4;
    L.colsum_a = off; off = up(off + rows);
    L.colsum_b = off; off = up(off + rows);
    L.absum = off; off = up(off + rows);
    L.zsum = off; off = up(off + (size_t)L.Npad * 4);
    L.b0 = off; off = up(off + (size_t)L.Npad * 4);
    L.barrier = off; off = up(off + 256);
    L.zero_bytes = off;
    L.fmax = off; off = up(off + (size_t)(T + 1) * L.Npad * 4);
    L.logz_a = off; off = up(off + (size_t)L.Npad * 4);
    L.logz_b = off; off = up(off + (size_t)L.Npad * 4);
    L.lz = off; off = up(off + (size_t)(T + 1) * L.Npad * 4);
    L.lnorm = off; off = up(off + (size_t)L.Npad * 8);
    L.bh = off; off = up(off + (size_t)2 * S * L.Npad * 4);
    L.total = off;
    return L;
}

int LaunchFrameMax(const void *y, int y_dtype, long sn, long st, int N, int T, int V, const int *len, float *fmax,
                   int Npad, cudaStream_t stream) {
    const long rows = (long)N * T;
    if (rows == 0) return 0;
    const int wpb = 8;
    frame_max_kernel<<<(unsigned)((rows + wpb - 1) / wpb), wpb * 32, 0, stream>>>(y, y_dtype, sn, st, N, T, V, len, fmax, Npad);
    CountLaunch();
    return (int)cudaGetLastError();
}

int LaunchFrameLse(const void *y, int y_dtype, long sn, long st, int N, int T, int V, const int *len, float *fmax,
                   float *lz, double *lnorm, int Npad, cudaStream_t stream) {
    const long rows = (long)N * T;
    if (rows == 0) return 0;
    const int wpb = 8;
    frame_lse_kernel<<<(unsigned)((rows + wpb - 1) / wpb), wpb * 32, 0, stream>>>(y, y_dtype, sn, st, N, T, V, len, fmax, lz, Npad);
    lnorm_kernel<<<N, 32, 0, stream>>>(lz, len, N, Npad, lnorm);
    CountLaunch(2);
    return (int)cudaGetLastError();
}

int LaunchLogitGrad(const void *z, int z_dtype, long sn, long st, int N, int T, int V, const int *len, const float *lz,
                    int Npad, float *grad, long gsn, long gst, cudaStream_t stream) {
    const long rows = (long)N * T;
    if (rows == 0) return 0;
    const int wpb = 8;
    logit_grad_kernel<<<(unsigned)((rows + wpb - 1) / wpb), wpb * 32, 0, stream>>>(z, z_dtype, sn, st, N, T, V, len, lz, Npad, grad, gsn, gst);
    CountLaunch();
    return (int)cudaGetLastError();
}

int LaunchDen(bool backward, const DeviceGraph &g, DenParams &p, cudaStream_t stream, std::string *err) {
    const DevicePass &pass = backward ? g.bwd : g.fwd;
    p.arcs = pass.arcs; p.chunk_state = pass.chunk_state; p.chunk_arc = pass.chunk_arc;
    p.chunk_pair = pass.chunk_pair; p.cta_labels = pass.cta_labels; p.w1 = backward ? pass.w1 : nullptr;
    p.own_c = pass.own_c; p.own = g.own_rows ? 1 : 0;
    DenHooks hooks = g.hooks;   // (a copy: a launch without a tensor map is chosen as without TMA)
    DenLaunch L;
    if (!ChooseDenLaunch(g.shape, p.Npad, backward, g.max_smem_optin, hooks, &L, err)) return 1;
    const size_t rows = backward ? (size_t)2 * g.S : (size_t)p.a_frames * g.S;   // TMA row coordinates stay below kOobRow
    if (L.tier == kTierSmall && rows >= kOobRow) { *err = "den: small-batch kernels: gather table of " + std::to_string(rows) + " rows"; return 1; }
    if (L.tier == kTierStreamed && !(rows < kOobRow && EncodeRowTensorMap(&p.tmap, p.bh, rows, p.Npad, 32 * L.U))) {
        hooks.no_tma = true;
        if (!ChooseDenLaunch(g.shape, p.Npad, backward, g.max_smem_optin, hooks, &L, err)) return 1;
    }
    p.tq = L.tier == kTierStreamed ? pass.tq : nullptr;
    p.tile_rows = L.tile_rows; p.gacc_rows = L.gacc_rows;
    p.ring_off = (int)L.ring_off; p.bar_off = (int)L.bar_off; p.abar_off = (int)L.abar_off; p.aring_off = (int)L.aring_off;
    return LaunchCoop(DenKernel(backward, L, g.shape.n_hubs > 0), p, g.n_ctas, L.total, stream, err);
}

int LaunchDenGradNormalize(float *grad, long gsn, long gst, const float *absum, const int *len, int N, int Npad,
                           int T, int V, float scale, cudaStream_t stream) {
    if ((long)N * T == 0) return 0;
    den_grad_normalize_kernel<<<(unsigned)((long)N * T), 128, 0, stream>>>(grad, gsn, gst, absum, len, N, Npad, T, V, scale);
    CountLaunch();
    return (int)cudaGetLastError();
}

}  // namespace ccb
