// Shared device helpers and the internal host-side launch interface (not part of the C ABI).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <memory>
#include <string>

#include "../../include/ctc_crf_b200.h"
#include "den_launch.h"

namespace ccb {

// ------------------------------------------------------------------------------------------------
// Device copy of the den plan (one per GPU listed in Init()).
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kOobRow = 0x40000000u;   // a TMA row coordinate no gather table reaches (tables are limited to 2^30 rows)

struct DevicePass {
    Arc *arcs = nullptr;
    int *chunk_state = nullptr;
    int *chunk_arc = nullptr;
    int *chunk_pair = nullptr;
    int *cta_labels = nullptr;
    float *w1 = nullptr;      // backward pass: second weight per slot
    float *own_c = nullptr;   // [2S + 4] own-row coefficients of this pass (DenPlan::own_fwd / own_bwd)
    // streamed-arc tier (DenGraphShape::streamed_quads, else null): the backward quads as the TMA kernel stages them, 3
    // 16-byte words per quad {row coordinate 0..3}{w0 0..3}{w1 0..3}
    uint4 *tq = nullptr;
};

struct DeviceGraph {
    bool loaded = false;
    int device = -1;
    int S = 0, P = 0, start = 0, num_labels = 0;   // S states, P pairs (gather-table rows S..S+P-1 = virtual pair-sum rows)
    int scale_exp = 56;
    int n_ctas = 0;
    DenGraphShape shape;   // what the kernel launch is chosen on (den_launch.h)
    int *state_label = nullptr;
    int *state_pos = nullptr;
    float *final_lin = nullptr;
    DevicePass fwd, bwd;
    Arc *start_arcs = nullptr;   // out-arcs of the start state
    int n_start_arcs = 0;
    int *hub_states = nullptr;   // states whose forward row is accumulated from parts (shape.n_hubs)
    float start_final = 0.f;
    int max_smem_optin = 0;
    DenHooks hooks;        // test hooks, read ONCE at Init (never on the per-call path)
    // batches of <= 16 utterances run the small-batch kernels (rows of 16 floats): SmallBatchOk, decided once at Init
    bool small_ok = false;
    bool own_rows = false;     // DenPlan::own_rows: own-row coefficients instead of own-row arcs (DevicePass::own_c)
    // the posterior sampler's in-arc CSR (DenPlan::in_off / in_src / in_w): uploaded by the first sampling call on the device,
    // from the host copy Init keeps, so that callers who never sample do not hold it in device memory
    std::shared_ptr<const DenPlan> host_plan;
    int *in_off = nullptr, *in_src = nullptr;
    float *in_w = nullptr;
    // the beam search's out-arc CSR (DenPlan::out_off / out_dst / out_w), likewise uploaded by the first crf=1 beam search on
    // the device, after CheckCtcShape has passed; ctc_shape caches that check (-1 not run yet, 0 passed, 1 failed: ctc_shape_err)
    int *out_off = nullptr, *out_dst = nullptr;
    float *out_w = nullptr;
    int ctc_shape = -1;
    std::string ctc_shape_err;
};

// Kernel parameter block shared by the two persistent den kernels (passed as a __grid_constant__ kernel parameter: the TMA
// descriptor inside it is read by the hardware straight from parameter memory and must sit on a 64-byte boundary).
struct alignas(64) DenParams {
    // TMA view of the backward gather table (the beta ping-pong) as a 2-D tensor [rows][Npad] of fp32 with a box of one
    // row x (32 * utterances per lane) columns; used by the streamed-arc tier only
    CUtensorMap tmap;
    // Byte offsets in dynamic shared memory (DenLaunch) of the streamed-arc tier's arc-ring mbarriers, the row rings and their
    // mbarriers.  (Kept at these offsets: shifting the pointers below by 8 bytes makes ptxas spill in several variants.)
    int abar_off;
    int ring_off;
    int bar_off;
    // graph
    const Arc *arcs;
    const float *w1;      // backward pass only
    const int *chunk_state;
    const int *chunk_arc;
    const int *chunk_pair;
    const int *cta_labels;
    const int *state_label;
    const int *state_pos;
    const uint4 *tq;          // streamed-arc tier: the pass's transposed quads in global memory (DevicePass::tq)
    int aring_off;            // ... byte offset in dynamic shared memory of the per-warp rings they flow through
    const float *final_lin;
    const Arc *start_arcs;
    int n_start_arcs;
    const int *hub_states;
    int n_hubs;
    int S, num_pairs, start, n_warps;
    int scale_exp;        // column sums are renormalised to ~2^scale_exp (DenPlan::scale_exp)
    float start_final;
    // problem
    const void *y;        // (N,T,V) log-probs, fp32, bf16 or fp16
    int y_dtype;          // CCB_DTYPE_* code of y (load_y)
    long sn, st;          // element strides of y
    int N, Npad, Tmax, V;
    const int *len;       // [N] device
    // workspaces
    float *alpha;         // [(Tmax+3)][S][Npad] scaled-linear alpha spill; the pair-sum rows of frame t are parked in frame t+2
    // Frame addressing of `alpha` (den_kernels.cu alpha_pos): frame t sits at position t - a_base, modulo a_ring when
    // a_ring > 0.  The full spill is a_base = a_ring = 0, the identity.  a_frames = positions the buffer holds.
    int a_base, a_ring, a_frames;
    // Checkpointed denominator (DESIGN.md "Checkpointed alpha"): ckpt_mode 0 = full spill; 1 = first forward pass on a
    // ring, storing the real rows of every ckpt_k-th frame in `ckpt` and logZ frame by frame; 2 = recompute of the frames
    // (t_lo, t_hi] from the checkpoint of frame t_lo, reading colsum_a and writing no logZ
    int ckpt_mode, ckpt_k;
    float *ckpt;          // [ceil(Tmax/ckpt_k)][S][Npad] real rows of frames 0, K, 2K, ...
    int t_lo, t_hi;       // frames (t_lo, t_hi] walked by this launch (one launch per pass: 0, Tmax)
    double *runlog_b;     // [Npad] backward log-scale books carried from one segment launch to the next
    float *bh;            // [2][S][Npad]          backward ping-pong (emission-weighted beta)
    float *colsum_a;      // [(Tmax+2)][Npad]
    float *colsum_b;      // [(Tmax+2)][Npad]
    float *absum;         // [(Tmax+2)][Npad]      sum_q alpha_t(q) beta_t(q)
    float *zsum;          // [Npad]
    float *b0;            // [Npad]
    const float *fmax;    // [Tmax][Npad]          per-frame max of y (emission shift)
    unsigned *barrier;    // grid barrier counter (zeroed before launch)
    float *logz;          // [N] out (forward: logZ from alpha; backward: logZ from beta)
    const float *own_c;   // [2S + 4] own-row coefficients of this pass (den_graph.h DenPlan::own_rows), used when own != 0
    int own;
    int own_off;          // byte offset in dynamic shared memory of the on-chip own rows (DenLaunch::own_smem; OWN_SMEM kernels)
    const double *lnorm;  // [N] or null: sum_t log-normaliser of raw logits, subtracted from logZ (raw-logit entry)
    // gradient (backward)
    float *grad;          // raw accumulation target, element (n,t,k) at n*gsn + t*gst + k
    long gsn, gst;
    int gacc_rows;        // rows of the shared-memory label accumulator (0 = direct global atomics)
    int tile_rows;        // max rows (states) owned by one CTA: size of the shared-memory row metadata
    // optional per-warp timeline (profiling aid, normally null)
    unsigned long long *timeline;
    int tl_step0, tl_steps;
};

// workspace carving (all offsets in bytes, 256-aligned)
struct DenAuxLayout {
    int Npad = 0;
    size_t colsum_a = 0, colsum_b = 0, absum = 0, zsum = 0, b0 = 0, barrier = 0, zero_bytes = 0;
    size_t fmax = 0, bh = 0, logz_a = 0, logz_b = 0, lz = 0, lnorm = 0, total = 0;
};
// Lane padding of a batch: whole 32-lane groups carrying 1, 2 or 4 utterances per lane; batches of <= 16 utterances on a
// graph that supports the small-batch kernels (DeviceGraph::small_ok) use 16-float rows instead (den_kernels.cu SMALL).
inline int PadLanes(int N, bool small_ok) {
    // (16-float rows even for N <= 8: the row copies are bound by their count, not by their bytes)
    if (small_ok && N <= 16) return 16;
    int g = (N + 31) / 32;
    if (g >= 3) g = (g + 3) / 4 * 4;   // lanes carry 1, 2 or 4 utterances each
    return g * 32;
}
DenAuxLayout MakeDenAuxLayout(int S, int N, int T, bool small_ok);

// host launchers; return cudaError_t-compatible int (0 = ok) and fill *err
int LaunchFrameMax(const void *y, int y_dtype, long sn, long st, int N, int T, int V, const int *len, float *fmax,
                   int Npad, cudaStream_t stream);
int LaunchFrameLse(const void *y, int y_dtype, long sn, long st, int N, int T, int V, const int *len, float *fmax,
                   float *lz, double *lnorm, int Npad, cudaStream_t stream);
int LaunchLogitGrad(const void *z, int z_dtype, long sn, long st, int N, int T, int V, const int *len, const float *lz,
                    int Npad, float *grad, long gsn, long gst, cudaStream_t stream);
// Checkpointed alpha workspace for K = ckpt_k (0: the full spill): frame positions of the first pass's ring / of one
// segment, then the checkpoints, then the backward pass's carried log-scales (see den_kernels.cu alpha_pos)
constexpr int kAlphaRing = 4;
inline int CkptK(int T, int K) { return K < T ? K : T; }
inline int CkptSegFrames(int T, int K) { const int k = CkptK(T, K); return (k + 1 > kAlphaRing ? k + 1 : kAlphaRing) + 2; }
inline int CkptCount(int T, int K) { const int k = CkptK(T, K); return (T + k - 1) / k; }
// one persistent den pass (the forward or the backward recursion) with the launch den_launch.h chooses
int LaunchDen(bool backward, const DeviceGraph &g, DenParams &p, cudaStream_t stream, std::string *err);
int LaunchDenGradNormalize(float *grad, long gsn, long gst, const float *absum, const int *len, int N, int Npad,
                           int T, int V, float scale, cudaStream_t stream);
// zero_inf: an utterance whose cost is not finite (log p, or logz[n] when logz is given, not finite) gets zero gradient rows
// t < len[n] -- written over whatever the den passes left there -- instead of its occupancies
int LaunchCtc(const void *y, int y_dtype, long sn, long st, int N, int T, int V, const int *labels,
              const int *label_off, const int *label_len, const int *len, int max_label_len, int blank,
              float *alpha_ws, float *grad, long gsn, long gst, float grad_scale, float *logp,
              const double *lnorm, cudaStream_t stream, std::string *err, int overwrite = 0, int Tfull = 0,
              const float *logz = nullptr, int zero_inf = 0);
// forward-only numerator: logp[n] = log p(l_n | x_n) (normalised by lnorm[n] when given) from the alpha chains alone, one
// CTA per utterance, no workspace; infeasible utterances get -inf
int LaunchCtcLogp(const void *y, int y_dtype, long sn, long st, int N, int T, int V, const int *labels,
                  const int *label_off, const int *label_len, const int *len, int max_label_len, int blank, float *logp,
                  const double *lnorm, cudaStream_t stream, std::string *err);
// The loss assembly: cost[n] = -logp[n] (CTC) or logz[n] - (1+lamb) logp[n] (CTC-CRF), in fp64; loss[0] = scale * sum_n cost[n].
// costs (N floats, may be null) receives every cost; zero_inf sets the costs that are not finite to 0 before both.
int LaunchSumScale(const float *logp, int N, float scale, float *loss, cudaStream_t stream, float *costs = nullptr,
                   int zero_inf = 0);
int LaunchCtcViterbi(const void *y, int y_dtype, long sn, long st, int N, int T, int V, const int *labels,
                     const int *label_off, const int *label_len, const int *len, int max_label_len, int blank,
                     unsigned char *bp_ws, int *align, float *score, cudaStream_t stream, std::string *err);
int LaunchAssembleLoss(const float *logz, const float *logp, int N, float lamb, float scale, float *loss,
                       cudaStream_t stream, float *costs = nullptr, int zero_inf = 0);
// Several label sequences per utterance.  Sequence m (of M, grouped by utterance) is scored against logits row seq_row[m];
// seq_pos[m] is its index in the caller's order; the sequences of utterance n are seq_off[n] .. seq_off[n+1]-1.
// The numerator's alpha (|| beta) chains over the M sequences: logp[m], and the cells of sequence m in alpha_ws (null: none).
int LaunchCtcSeqs(const void *y, int y_dtype, long sn, long st, int M, int T, int V, const int *labels,
                  const int *label_off, const int *label_len, const int *len, const int *seq_row, int max_label_len,
                  int blank, float *alpha_ws, bool want_beta, float *logp, const double *lnorm, cudaStream_t stream,
                  std::string *err);
// The occupancies of every sequence of an utterance summed into its rows, once: out = W_n den + num_coef sum_m w_m gamma_m
// (ctc_kernels.cu ctc_gamma_seqs_kernel); every row t < Tfull of the N utterances is written.
int LaunchCtcGammaSeqs(const void *y, int y_dtype, long sn, long st, int N, int T, int Tfull, int V, const int *labels,
                       const int *label_off, const int *label_len, const int *len, const int *seq_off, const int *seq_pos,
                       int max_label_len, int blank, float *alpha_ws, const float *w, float w_scale, float num_coef,
                       const float *den, const float *logz, int zero_inf, float *out, long gsn, long gst, cudaStream_t stream,
                       std::string *err);
// costs[seq_pos[m]] = logz[seq_row[m]] - (1+lamb) logp[m] (logz = null: -logp[m]); loss[0] = scale * sum_m cost
int LaunchSeqCosts(const float *logz, const float *logp, const int *seq_row, const int *seq_pos, int M, float lamb, float scale,
                   float *loss, float *costs, int zero_inf, cudaStream_t stream);
int LaunchCtcViterbiSeqs(const void *y, int y_dtype, long sn, long st, int M, int T, int V, const int *labels,
                         const int *label_off, const int *label_len, const int *len, const int *seq_row, const int *seq_pos,
                         int max_label_len, int blank, unsigned char *bp_ws, int *align, float *score, cudaStream_t stream,
                         std::string *err);
// out[n][t][:] = w[n] * grad[n][t][:] for t < len[n], 0 beyond (grad not read there); out in the CCB_DTYPE_* out_dtype
int LaunchGradRowsScale(const float *grad, const float *w, const int *len, int N, int T, int V, void *out, int out_dtype,
                        cudaStream_t stream);
void CountLaunch(int n = 1);
// Posterior sampler (den_sample.cu) over alpha frames held at positions t - a_base of `alpha` ([pos][S][Npad]).
// Workspace: a SampleRec per (utterance, sample), then per utterance S doubles of the final-state prefix sum.
struct SampleRec {
    int q;          // state at the frame the walk has reached
    int last_lab;   // label of that frame (-1 before the first), for the collapse
    int ntok;       // tokens written so far, last one first
    int status;     // kSamplePending / kSampleWalking / kSampleDead
    double score;   // sum of y + log w (+ log final) of the frames walked so far
    double pad;
};
constexpr int kSamplePending = 0, kSampleWalking = 1, kSampleDead = 2;
size_t SampleWsBytes(int N, int K, int S);
// Final-state prefix sums of the utterances whose length lies in (t_lo, t_hi]
int LaunchSampleFinalPrefix(const float *alpha, int a_base, int S, int Npad, const float *final_lin, const int *len, int N,
                            int t_lo, int t_hi, void *sample_ws, int K, cudaStream_t stream);
// The backward walk over frames (t_lo, t_hi] for all K samples of the N utterances; first: this is the first launch of the
// call (initialise the records), t_lo == 0: the last (write the outputs)
int LaunchSampleWalk(const DeviceGraph &g, const void *y, int y_dtype, long sn, long st, int N, int T, int Tmax, int Npad,
                     const int *len, const float *alpha, int a_base, int t_lo, int t_hi, bool first, int K,
                     unsigned long long seed, int n_base, const float *logz, void *sample_ws, int *tokens, int *lengths,
                     int *align, float *path_logp, cudaStream_t stream);
// CTC prefix beam search (beam_search.cu): one CTA per utterance, one launch for the batch.  g: the den graph for crf mode,
// null for plain CTC.  Workspace: per utterance the trie (B*T + 1 nodes) and its hash table.
constexpr int kBeamMax = 128;
constexpr int kBeamMaxV = 8192;
size_t BeamWsBytes(int N, int T, int B);
// A token n-gram LM's tables on one device (ngram.h NGramHost), for shallow fusion into the plain-mode search
struct NGramDev {
    const int *tok2word = nullptr, *root_dst = nullptr, *arc_off = nullptr, *arc_word = nullptr, *arc_dst = nullptr,
              *back = nullptr;
    const float *root_p = nullptr, *arc_p = nullptr, *bow = nullptr;
    int bos = 0, eos = 0;
};
// lm null: the search without an LM; else every extension p -> p+c adds alpha ln P(c | p) + beta to the candidate's rank
int LaunchBeamSearch(const DeviceGraph *g, const void *y, int y_dtype, int N, int T, int V, const int *len, int B, int topn,
                     void *ws, int *tokens, int *lengths, int *timesteps, float *scores, cudaStream_t stream,
                     const NGramDev *lm = nullptr, double alpha = 0.0, double beta = 0.0);
// The n-gram LM's rows for the fused RNN-T step (rnnt_decode.cu): one CTA per slot of N*B, W the LM's word count; its
// dynamic shared memory is NgramSlotRowsSmemBytes(W)
size_t NgramSlotRowsSmemBytes(int W);
int LaunchNgramSlotRows(const NGramDev &lm, int W, int N, int B, int V, const int *parent, const int *token,
                        const int *state_in, int *state_out, float *rows, cudaStream_t s);
// The rows of a weighted LM mix for the fused RNN-T step (rnnt_decode.cu): one CTA per slot of N*B.  Member i is an n-gram
// LM (rows null: its tables, word count W and (N, B) int32 state arrays) or a neural LM (its (N*B, V) row block in the
// CCB_DTYPE_* code dtype); w is its weight.  W: the largest n-gram word count (0 without one); the dynamic shared memory is
// LmMixSlotRowsSmemBytes(W, V)
constexpr int kLmMixMax = 8;
struct LmMixMember {
    NGramDev lm;
    const int *state_in = nullptr;
    int *state_out = nullptr;
    const void *rows = nullptr;
    int dtype = 0, W = 0;
    double w = 0.0;
};
struct LmMixDev {
    int K = 0;
    LmMixMember m[kLmMixMax];
};
size_t LmMixSlotRowsSmemBytes(int W, int V);
int LaunchLmMixSlotRows(const LmMixDev &mix, int W, int N, int B, int V, const int *parent, const int *token, float *rows,
                        cudaStream_t s);
// Sentence scores under an n-gram LM (ngram_score.cu), one launch: R rows of token ids (row stride ids_stride, U columns
// read up to each row's length), each row's last target (row stride last_stride), lengths (null: U); *_i64 selects int64
// over int32.  bos_word: the word id of <s>; order: the LM's order.  out: (R,) fp32, NaN for a row with a bad token or length.
struct NGramScoreArgs {
    NGramDev lm;
    int V = 0, order = 0, bos_word = 0, R = 0, U = 0;
    const void *ids = nullptr, *last = nullptr, *lens = nullptr;
    long ids_stride = 0, last_stride = 0;
    int ids_i64 = 0, last_i64 = 0, lens_i64 = 0;
    float *out = nullptr;
};
int LaunchNgramScore(const NGramScoreArgs &a, cudaStream_t s);
// A decoding graph's tables on one device (wfst.h WfstHost), for the TLG Viterbi beam search (wfst_decode.cu)
struct WfstDev {
    const int *arc_off = nullptr, *eps_off = nullptr, *dst = nullptr, *tok = nullptr, *olabel = nullptr, *fid = nullptr,
              *src = nullptr, *lay = nullptr, *level = nullptr;
    const float *w = nullptr, *final_cost = nullptr;
    int S = 0, start = 0, L = 0, E = 0, max_out = 0;
};
constexpr int kWfstMaxActive = 1 << 20;
constexpr int kWfstMaxV = 8192;
// Workspace of N utterances of T frames at max_active K: per utterance two state hashes sized from K, the largest emitting
// out-degree and the largest epsilon closure (never more states than the graph has), and the (T+1) x K records of L+1 arcs
size_t WfstWsBytes(const WfstDev &g, int N, int T, int K);
int LaunchWfstDecode(const WfstDev &g, const void *y, int y_dtype, int N, int T, int V, const int *len, float acwt, float lmwt,
                     float wip, float beam, int K, void *ws, int *words, int *num_words, int *align, float *ac_logp,
                     float *graph_cost, float *cost, int *reached_final, cudaStream_t stream);
// The RNN-T (CTCT = false) and CTC-T (CTCT = true) losses (rnnt_kernels.cu); lengths and labels are device pointers.
// Over the joint tensor: the forward runs the prep, row and alpha (|| beta when want_beta) passes; the backward the gradient
// pass over the same workspace of WsBytes(N, rows) bytes.  Of the LogAdd joiner, from f (N, Tmax, V) and g (N, Umax+1, V):
// the forward runs the prep, row maxima, normaliser GEMM, underflow fix-up and alpha (|| beta) passes; the backward the cell
// weights and the two gradient GEMMs over the same workspace of SimpleWsBytes(N, Tmax, Umax) bytes.
template <bool CTCT> struct TransducerLoss {
    static size_t WsBytes(int N, long long rows);
    static int Forward(const void *x, int dtype, int from_logits, int compact, int N, long long rows, int V, int Tmax, int Umax,
                       const int *labels, long long n_labels, const int *lx, const int *ly, int blank, int want_beta, void *ws,
                       float *costs, float *costs_beta, cudaStream_t s);
    static int Backward(const void *x, int dtype, int from_logits, int N, long long rows, int V, const int *labels, int blank,
                        void *ws, const float *w, void *grad, cudaStream_t s);
    static size_t SimpleWsBytes(int N, int Tmax, int Umax);
    static int SimpleForward(const void *f, const void *g, int dtype, int N, int Tmax, int Umax, int V, const int *labels,
                             const int *lx, const int *ly, int blank, int want_beta, void *ws, float *costs, cudaStream_t s);
    static int SimpleBackward(const void *f, const void *g, int dtype, int N, int Tmax, int Umax, int V, const int *labels,
                              int blank, void *ws, const float *w, void *grad_f, void *grad_g, cudaStream_t s);
};
// Transducer beam search (rnnt_decode.cu): init, one step per frame, finish; one CTA per utterance each
constexpr int kRnntBeamMaxV = 1 << 24;
size_t RnntBeamWsBytes(int N, int T, int B);
int LaunchRnntBeamInit(int N, int T, int B, void *ws, int *parent, int *token, int *node, double *score, cudaStream_t s);
int LaunchRnntBeamStep(const void *rows, const void *enc, int dtype, int mode, int N, int T, int B, int V, int t,
                       const int *len, int blank, void *ws, int *parent, int *token, int *node, double *score, cudaStream_t s);
int LaunchRnntBeamFinish(int N, int T, int B, int nbest, const void *ws, const int *node, const double *score, int *tokens,
                         int *lengths, float *scores, cudaStream_t s);
// the step with LM / ILM fusion (either row block may be null, not both); lm_part (N, B) fp64 read and written
int LaunchRnntBeamStepFused(const void *rows, const void *enc, int dtype, int mode, int N, int T, int B, int V, int t,
                            const int *len, int blank, void *ws, int *parent, int *token, int *node, double *score,
                            const void *lm_rows, int lm_dtype, double alpha, double beta, const void *ilm_rows, int ilm_dtype,
                            double ilm_weight, double *lm_part, cudaStream_t s);
// CTC-T beam search (ctct_decode.cu): init and one step per frame over a workspace that starts with the transducer beam
// search's tries (same stride), so that LaunchRnntBeamFinish finishes it
size_t CtctBeamWsBytes(int N, int T, int B);
int LaunchCtctBeamInit(int N, int T, int B, void *ws, int *parent, int *token, int *node, double *score, cudaStream_t s);
int LaunchCtctBeamStep(const void *rows, const void *enc, int dtype, int mode, int N, int T, int B, int V, int t,
                       const int *len, int blank, void *ws, int *parent, int *token, int *node, double *score, cudaStream_t s);
// gather.sum of the joiner and its backward; ws: GatherWsBytes(N) bytes of per-utterance offsets
size_t GatherWsBytes(int N);
int LaunchGatherSum(const void *a, const void *b, int dtype, int N, long long rows_out, int H, const int *la, const int *lb,
                    void *ws, void *out, cudaStream_t s);
int LaunchGatherSumBackward(const void *g, int dtype, int N, long long rows_a, long long rows_b, int H, const int *la,
                            const int *lb, void *ws, void *grad_a, void *grad_b, cudaStream_t s);

// ------------------------------------------------------------------------------------------------
// device helpers
// ------------------------------------------------------------------------------------------------
#ifdef __CUDACC__
// Element idx of the logits as float.  dtype is a CCB_DTYPE_* code: fp32 is read as is; bf16 and fp16 share one 16-bit
// load and differ only in the convert (callers accept no other code).
__device__ __forceinline__ float load_y(const void *y, int dtype, long idx) {
    if (dtype == CCB_DTYPE_F32) return __ldg(reinterpret_cast<const float *>(y) + idx);
    const unsigned short h = reinterpret_cast<const unsigned short *>(y)[idx];
    return dtype == CCB_DTYPE_BF16 ? __bfloat162float(__ushort_as_bfloat16(h)) : __half2float(__ushort_as_half(h));
}

// The inverse of load_y: v stored as element idx of a buffer in the CCB_DTYPE_* code `dtype` (round to nearest even)
__device__ __forceinline__ void store_y(void *out, int dtype, long idx, float v) {
    if (dtype == CCB_DTYPE_F32) { reinterpret_cast<float *>(out)[idx] = v; return; }
    reinterpret_cast<unsigned short *>(out)[idx] = dtype == CCB_DTYPE_BF16 ? __bfloat16_as_ushort(__float2bfloat16_rn(v))
                                                                           : __half_as_ushort(__float2half_rn(v));
}

__device__ __forceinline__ void red_release_add_u32(unsigned *p, unsigned v) {
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Grid-wide barrier for a co-resident (cooperatively launched) grid.  `target` is the value the
// monotonically increasing counter reaches once every CTA has arrived at this barrier.
// Arrive with a release reduction, poll with relaxed loads (an acquire load would invalidate L1 on every poll),
// then one acquire fence before the CTA is released.
__device__ __forceinline__ void grid_barrier(unsigned *counter, unsigned target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        red_release_add_u32(counter, 1u);
        unsigned v;
        do {
            asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
        } while (v < target);
        asm volatile("fence.acq_rel.gpu;" ::: "memory");
    }
    __syncthreads();
}

// The same barrier in two halves: work placed between them (by any thread of the CTA) overlaps the barrier latency.
// Only writes made BEFORE the arrive are guaranteed visible to the other CTAs after their wait; writes made in between
// are ordered by the NEXT barrier's release (use them for data nobody reads in the next frame).
__device__ __forceinline__ void grid_barrier_arrive(unsigned *counter) {
    __syncthreads();
    if (threadIdx.x == 0) red_release_add_u32(counter, 1u);
}
__device__ __forceinline__ void grid_barrier_wait(unsigned *counter, unsigned target) {
    if (threadIdx.x == 0) {
        unsigned v;
        do {
            asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
        } while (v < target);
        asm volatile("fence.acq_rel.gpu;" ::: "memory");
    }
    __syncthreads();
}

// log-semiring add in fp32 (numerator only), same formula as den_calculate.cu:28-35 / ctc_helper.h.  The operands
// are kept relative to a per-frame offset (|values| stay small), so the hardware ex2/lg2 approximations
// (abs. error ~1e-7 here) are as accurate as the libm versions were on the reference's un-normalised values.
__device__ __forceinline__ float log_add(float a, float b) {
    const float m = fmaxf(a, b);
    if (m == -INFINITY) return m;
    return m + __logf(1.f + __expf(-fabsf(a - b)));   // exp(-inf) = 0 covers a one-sided -inf
}
#endif

}  // namespace ccb
