// Exact samples from the CTC-CRF posterior p(path | x) over the den graph: forward filtering, backward sampling.
//
// The filtering half is the den forward pass: its alpha spill holds alpha_t(q) for every frame, state and utterance, scaled
// by a power of two per (frame, utterance) column (den_kernels.cu), and only ratios inside one column are used here.  The
// backward half (DESIGN.md §7 "Posterior samples"):
//   * the state of the last frame t = len is drawn with probability ~ alpha_len(q) final(q): a per-utterance prefix sum
//     (sample_final_prefix_kernel, O(S) per utterance, not per sample), then a binary search per sample;
//   * then, frame by frame down to t = 1, a predecessor p of the current state q with probability ~ alpha_{t-1}(p) w_pq
//     (sample_walk_kernel: one warp per (utterance, sample); the lanes take q's in-arcs in chunks of 32).
// Every draw is an inverse CDF in fp64 with ONE uniform: the first arc whose running sum exceeds u * total.  The uniform of
// the draw that picks the state of frame t is Philox4x32-10 keyed by the call's seed at counter (t, sample, utterance, 0),
// written out here (not cuRAND's state API) so that the numpy restatement in tests/test_sample_dispatch.py reproduces every
// uniform bit for bit, and so that the samples of an utterance do not depend on how the batch was sliced or on the other utterances in it.
#include <cmath>

#include "common.cuh"

namespace ccb {

namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kWalkThreads = 128;     // 4 (utterance, sample) walks per CTA
constexpr int kPrefixThreads = 512;

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
        const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    return c;
}

// u in [0, 1) with 53 random bits: words 0 and 1 of the Philox block at counter (frame, sample, utterance, 0)
__device__ __forceinline__ double draw_uniform(unsigned long long seed, int frame, int sample, int utt) {
    const uint4 x = philox4x32_10(make_uint4((uint32_t)frame, (uint32_t)sample, (uint32_t)utt, 0u), (uint32_t)seed,
                                  (uint32_t)(seed >> 32));
    return ((double)(x.x >> 5) * 67108864.0 + (double)(x.y >> 6)) * (1.0 / 9007199254740992.0);
}

// u * total, kept strictly below total (u * total rounds to total for u within 2^-53 of 1)
__device__ __forceinline__ double draw_target(double u, double total) {
    const double x = u * total;
    return x < total ? x : nextafter(total, 0.0);
}

__device__ __forceinline__ double warp_incl_scan(double v, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const double o = __shfl_up_sync(kFull, v, d);
        if (lane >= d) v += o;
    }
    return v;
}

// The weight of one arc of the draw: w * alpha_{t-1}(src) in fp64 (no product of two floats underflows there); zero, -0
// and NaN (a column the den pass could not scale) count as no weight.
__device__ __forceinline__ double arc_weight(float w, float a) {
    const double v = (double)w * (double)a;
    return v > 0.0 ? v : 0.0;
}

SampleRec *Records(void *ws) { return reinterpret_cast<SampleRec *>(ws); }
__host__ __device__ __forceinline__ size_t RecordBytes(int N, int K) {
    return ((size_t)N * (size_t)K * sizeof(SampleRec) + 255) & ~(size_t)255;
}

// prefix[n][q] = sum_{q' <= q} final(q') alpha_len(q'), fp64, for the utterances whose last frame lies in (t_lo, t_hi].
// Each thread sums a contiguous run of states, thread 0 chains the run totals, then every thread adds its offset: so the
// prefix never decreases, and a state at which it increases has a positive weight.
__global__ void __launch_bounds__(kPrefixThreads) sample_final_prefix_kernel(
        const float *alpha, int a_base, int S, int Npad, const float *final_lin, const int *len, int t_lo, int t_hi,
        double *prefix_all) {
    __shared__ double s_tot[kPrefixThreads];
    const int n = blockIdx.x;
    const int ln = len[n];
    if (!(ln > t_lo && ln <= t_hi)) return;
    const float *fr = alpha + (size_t)(ln - a_base) * (size_t)S * Npad + n;
    double *prefix = prefix_all + (size_t)n * S;
    const int per = (S + kPrefixThreads - 1) / kPrefixThreads;
    const int q0 = min(S, (int)threadIdx.x * per), q1 = min(S, q0 + per);
    double acc = 0.0;
    for (int q = q0; q < q1; ++q) {
        const float f = final_lin[q];
        if (f != 0.f) acc += arc_weight(f, fr[(size_t)q * Npad]);
        prefix[q] = acc;
    }
    s_tot[threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double off = 0.0;
        for (int i = 0; i < kPrefixThreads; ++i) { const double v = s_tot[i]; s_tot[i] = off; off += v; }
    }
    __syncthreads();
    const double off = s_tot[threadIdx.x];
    for (int q = q0; q < q1; ++q) prefix[q] = off + prefix[q];
}

struct WalkParams {
    const int *state_label, *in_off, *in_src;
    const float *in_w, *final_lin;
    int S, start;
    const void *y;
    int y_dtype;
    long sn, st;
    int N, T, Tmax, Npad;
    const int *len;
    const float *alpha;
    int a_base, t_lo, t_hi, first, K, n_base;
    unsigned long long seed;
    const float *logz;
    SampleRec *rec;
    const double *prefix;
    int *tokens, *lengths, *align;
    float *path_logp;
};

// One warp per (utterance, sample).  The record (state, score, collapse) lives in registers for the frames of this launch and
// in the workspace between launches (checkpointed alpha: one launch per segment, last segment first).  score, ntok and
// last_lab are kept by lane 0; q and status are the same in every lane.
__global__ void __launch_bounds__(kWalkThreads) sample_walk_kernel(const WalkParams P) {
    const int lane = threadIdx.x & 31;
    const long w = (long)blockIdx.x * (kWalkThreads / 32) + (threadIdx.x >> 5);
    if (w >= (long)P.N * P.K) return;
    const int n = (int)(w / P.K), k = (int)(w % P.K);
    const int utt = P.n_base + n;
    const int ln = P.len[n];
    int *const al = P.align + (size_t)w * P.T;
    int *const tok = P.tokens + (size_t)w * P.T;
    SampleRec r;
    if (P.first) {
        r.q = 0; r.last_lab = -1; r.ntok = 0; r.score = 0.0; r.pad = 0.0;
        r.status = (ln > 0 && ln <= P.Tmax) ? kSamplePending : kSampleDead;
        for (int t = max(ln, 0) + lane; t < P.T; t += 32) al[t] = -1;   // frames past the length
    } else {
        r = P.rec[w];
    }
    // the state of the last frame: prefix sum of alpha_len(q) final(q), binary search
    if (r.status == kSamplePending && ln > P.t_lo && ln <= P.t_hi) {
        const double *pre = P.prefix + (size_t)n * P.S;
        const double total = pre[P.S - 1];
        if (total > 0.0 && isfinite(total)) {
            const double target = draw_target(draw_uniform(P.seed, ln, k, utt), total);
            int lo = 0, hi = P.S - 1;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (pre[mid] > target) hi = mid; else lo = mid + 1;
            }
            r.q = lo;
            r.score = log((double)P.final_lin[lo]);
            r.status = kSampleWalking;
        } else {
            r.status = kSampleDead;
        }
    }
    if (r.status == kSampleWalking) {
        const size_t frame = (size_t)P.S * P.Npad;
        for (int t = min(ln, P.t_hi); t > P.t_lo; --t) {
            const int q = r.q;
            const int beg = P.in_off[q], end = P.in_off[q + 1];
            const int lab = P.state_label[q];
            if (lane == 0) {   // frame t-1 of the logits carries the label of the state of alpha frame t
                al[t - 1] = lab;
                r.score += (double)load_y(P.y, P.y_dtype, (long)n * P.sn + (long)(t - 1) * P.st + lab);
                if (lab != 0 && lab != r.last_lab) tok[r.ntok++] = lab;   // a new run of a token (the collapse, read backwards)
            }
            r.last_lab = lab;
            const float *ap = P.alpha + (size_t)(t - 1 - P.a_base) * frame + n;
            // pass 1: the total weight of q's in-arcs (chunk 0 stays in registers for pass 2)
            int src0 = 0;
            float w0 = 0.f;
            double v0 = 0.0;
            if (beg + lane < end) {
                src0 = P.in_src[beg + lane];
                w0 = P.in_w[beg + lane];
                v0 = arc_weight(w0, ap[(size_t)src0 * P.Npad]);
            }
            const double inc0 = warp_incl_scan(v0, lane);
            const double tot0 = __shfl_sync(kFull, inc0, 31);
            double total = tot0;
            unsigned pos = __ballot_sync(kFull, v0 > 0.0);
            int last = pos ? beg + 31 - __clz(pos) : -1;   // the last arc with weight: the draw's fall-back
            for (int c = beg + 32; c < end; c += 32) {     // hub states: more chunks
                double v = 0.0;
                if (c + lane < end) v = arc_weight(P.in_w[c + lane], ap[(size_t)P.in_src[c + lane] * P.Npad]);
                total += __shfl_sync(kFull, warp_incl_scan(v, lane), 31);
                pos = __ballot_sync(kFull, v > 0.0);
                if (pos) last = c + 31 - __clz(pos);
            }
            if (!(total > 0.0 && isfinite(total)) || last < 0) { r.status = kSampleDead; break; }
            const double target = draw_target(draw_uniform(P.seed, t - 1, k, utt), total);
            // pass 2: the first arc with weight whose running sum exceeds the target
            int pick = -1;
            unsigned hit = __ballot_sync(kFull, inc0 > target && v0 > 0.0);
            if (hit) {
                pick = beg + __ffs(hit) - 1;
            } else {
                double base = tot0;
                for (int c = beg + 32; c < end && pick < 0; c += 32) {
                    double v = 0.0;
                    if (c + lane < end) v = arc_weight(P.in_w[c + lane], ap[(size_t)P.in_src[c + lane] * P.Npad]);
                    const double inc = warp_incl_scan(v, lane);
                    hit = __ballot_sync(kFull, inc + base > target && v > 0.0);
                    if (hit) pick = c + __ffs(hit) - 1;
                    base += __shfl_sync(kFull, inc, 31);
                }
            }
            if (pick < 0) pick = last;
            r.q = P.in_src[pick];
            if (lane == 0) r.score += log((double)P.in_w[pick]);
        }
    }
    if (P.t_lo > 0) {   // more segments follow
        if (lane == 0) P.rec[w] = r;
        return;
    }
    // last launch: the outputs of this walk
    const int ntok = __shfl_sync(kFull, r.ntok, 0);
    const double score = __shfl_sync(kFull, r.score, 0);
    const bool ok = r.status == kSampleWalking && r.q == P.start;
    __syncwarp();
    if (ok) {
        for (int i = lane; i < ntok / 2; i += 32) {   // the tokens were written last one first
            const int a = tok[i], b = tok[ntok - 1 - i];
            tok[i] = b;
            tok[ntok - 1 - i] = a;
        }
        for (int t = ntok + lane; t < P.T; t += 32) tok[t] = -1;
    } else {
        for (int t = lane; t < P.T; t += 32) { tok[t] = -1; al[t] = -1; }
    }
    if (lane == 0) {
        P.lengths[w] = ok ? ntok : -1;
        P.path_logp[w] = ok ? (float)(score - (double)P.logz[n]) : -INFINITY;
    }
}

}  // namespace

size_t SampleWsBytes(int N, int K, int S) { return RecordBytes(N, K) + (size_t)N * (size_t)S * sizeof(double); }

int LaunchSampleFinalPrefix(const float *alpha, int a_base, int S, int Npad, const float *final_lin, const int *len, int N,
                            int t_lo, int t_hi, void *sample_ws, int K, cudaStream_t stream) {
    double *prefix = reinterpret_cast<double *>(reinterpret_cast<char *>(sample_ws) + RecordBytes(N, K));
    sample_final_prefix_kernel<<<N, kPrefixThreads, 0, stream>>>(alpha, a_base, S, Npad, final_lin, len, t_lo, t_hi, prefix);
    CountLaunch();
    return (int)cudaGetLastError();
}

int LaunchSampleWalk(const DeviceGraph &g, const void *y, int y_dtype, long sn, long st, int N, int T, int Tmax, int Npad,
                     const int *len, const float *alpha, int a_base, int t_lo, int t_hi, bool first, int K,
                     unsigned long long seed, int n_base, const float *logz, void *sample_ws, int *tokens, int *lengths,
                     int *align, float *path_logp, cudaStream_t stream) {
    WalkParams p;
    p.state_label = g.state_label; p.in_off = g.in_off; p.in_src = g.in_src; p.in_w = g.in_w; p.final_lin = g.final_lin;
    p.S = g.S; p.start = g.start;
    p.y = y; p.y_dtype = y_dtype; p.sn = sn; p.st = st;
    p.N = N; p.T = T; p.Tmax = Tmax; p.Npad = Npad; p.len = len;
    p.alpha = alpha; p.a_base = a_base; p.t_lo = t_lo; p.t_hi = t_hi; p.first = first ? 1 : 0; p.K = K; p.n_base = n_base;
    p.seed = seed; p.logz = logz;
    p.rec = Records(sample_ws);
    p.prefix = reinterpret_cast<const double *>(reinterpret_cast<const char *>(sample_ws) + RecordBytes(N, K));
    p.tokens = tokens; p.lengths = lengths; p.align = align; p.path_logp = path_logp;
    const long warps = (long)N * K;
    const long blocks = (warps + kWalkThreads / 32 - 1) / (kWalkThreads / 32);
    sample_walk_kernel<<<(unsigned)blocks, kWalkThreads, 0, stream>>>(p);
    CountLaunch();
    return (int)cudaGetLastError();
}

}  // namespace ccb
