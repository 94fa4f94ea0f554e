/*
 * ctc_crf_b200 -- C ABI of the H100-native CTC-CRF loss hot path (drop-in for thu-spmi/CAT src/ctc_crf).
 *
 * Plain C, no torch types: pointers, sizes, a cudaStream_t passed as void*.  All device pointers must
 * belong to the CUDA device that is current when the call is made (the reference has the same contract,
 * den_calculate.cu:436-438).  Citations are relative to /root/reference/src/ctc_crf.
 *
 * Section 1 keeps the exact names and signatures the reference's binding.cpp binds (binding.cpp:14-49 and
 * gpu_ctc/ctc.h:16-109), so the reference's own binding.cpp links against this library unchanged.
 * Section 2 is the fused entry the new autograd Function uses (SURVEY.md 8b "new fused entry").
 * Section 3 exposes the host-side den-graph plan for CPU-only tests.
 *
 * Error convention: section-1 den functions return void like the reference but never exit(); they record
 * an error retrievable with ccb_last_error().  Everything else returns 0 on success, non-zero on failure.
 */
#ifndef CTC_CRF_B200_H_
#define CTC_CRF_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------
 * Section 1 -- reference-compatible entry points
 * ---------------------------------------------------------------------------------------------- */

/* replaces den_calculate.cu:263-273 globals read by binding.cpp:14-15,77-78 (scratch sizing).
 * DEN_NUM_STATES is the state count *after* the loader's in-label state split (== the file's state
 * count for every T-compose-LM graph). */
extern int DEN_NUM_ARCS;
extern int DEN_NUM_STATES;

/* replaces Init / Release (binding.cpp:22-24, den_calculate.cu:288-425): load an OpenFst binary
 * vector/standard den graph, build the kernel plan, upload it to each listed GPU. */
void Init(const char *fst_name, int n_gpus, int *gpus);
void Release(int n_gpus, int *gpus);

/* replaces compute_alpha (binding.cpp:26-34, den_calculate.cu:427-451).
 *   alpha      : scratch, >= ccb_den_alpha_floats(batch_size, T) floats (OPAQUE layout: [t][state][lane]).
 *                The need is (T+3) frames of DEN_NUM_STATES-P rows of PadLanes(N) floats (lanes padded to 32, 64 or a multiple
 *                of 128; 16 for batches of <= 16 utterances on small graphs): binding.cpp's (T+1)*N*DEN_NUM_STATES covers it
 *                for N = 32, 64, 128, 256 ... but NOT for every other N (e.g. 96 -> 128 lanes).  When the caller's buffer is
 *                too small the library takes its own from the device's default memory pool, stream-ordered
 *                (cudaMallocAsync on `stream`: no device synchronisation), keeps it between calls and returns it in Release().
 *                Size the buffer with ccb_den_alpha_floats() to avoid the second allocation.
 *   logits     : (N,T,V) fp32 log-probs, contiguous
 *   input_lengths : (N,) int32 DEVICE
 *   loglikelihood : (N,) fp32 DEVICE out, logZ_den per utterance */
void compute_alpha(float *alpha, float *logits, const int batch_size, int T, const int alpha_size,
                   int logits_size, int *input_lengths, float *loglikelihood, void *stream);

/* replaces compute_beta_and_grad (binding.cpp:36-48, den_calculate.cu:453-481).
 *   grad_net : (N,T,V) fp32, PRE-ZEROED by the caller (ctc_crf/__init__.py:66); rows t < len get the
 *              denominator occupancies, rows t >= len stay untouched.
 *   beta / grad_storage : scratch of the reference's sizes; unused here (kept for signature parity).
 *   loglikelihood : (N,) out, logZ_den recomputed from the backward pass (== alpha_lld up to rounding). */
void compute_beta_and_grad(float *beta, const float *const alpha, const float *const logits,
                           const float *const alpha_lld, float *grad_storage, float *grad_net,
                           const int batch_size, const int T, const int beta_size, const int logits_size,
                           const int *const input_lengths, float *loglikelihood, void *stream);

/* replaces gpu_ctc/ctc.h:16-109 */
typedef enum {
    CTC_STATUS_SUCCESS = 0,
    CTC_STATUS_MEMOPS_FAILED = 1,
    CTC_STATUS_INVALID_VALUE = 2,
    CTC_STATUS_EXECUTION_FAILED = 3,
    CTC_STATUS_UNKNOWN_ERROR = 4
} ctcStatus_t;

struct ctcOptions {
    void *stream;     /* CUstream */
    int blank_label;
};

const char *ctcGetStatusString(ctcStatus_t status);

/* activations: (T,N,V) fp32 log-probs on the device; gradients: (T,N,V) pre-zeroed device buffer or NULL;
 * flat_labels / label_lengths / input_lengths / costs: HOST pointers; costs[n] = log p(l_n | x_n). */
ctcStatus_t compute_ctc_loss(const float *const activations, float *gradients, const int *const flat_labels,
                             const int *const label_lengths, const int *const input_lengths, int alphabet_size,
                             int minibatch, float *costs, void *workspace, struct ctcOptions options);
ctcStatus_t get_workspace_size(const int *const label_lengths, const int *const input_lengths,
                               int alphabet_size, int minibatch, struct ctcOptions options, size_t *size_bytes);

/* ------------------------------------------------------------------------------------------------
 * Section 2 -- fused entry and helpers (additions)
 * ---------------------------------------------------------------------------------------------- */
/* Logits dtype codes, the `dtype` argument of every section-2 entry that takes one: the (N,T,V) block is read in this type
 * and converted to fp32 element by element; the arithmetic and every output (loss, parts, gradient, score) stay fp32.  fp16
 * is what CAT's `--amp` encoder returns (torch.cuda.amp autocast); bf16 what a bf16 autocast returns.  Any other code fails
 * with a message.  Section 1 takes fp32 only, as the reference does. */
#define CCB_DTYPE_F32 0
#define CCB_DTYPE_BF16 1
#define CCB_DTYPE_F16 2

const char *ccb_last_error(void);            /* thread-local message of the last failure ("" if none) */
int ccb_den_loaded(int device);              /* 1 if Init() covered this device */
/* info[0..7] = file states, file arcs, states after the in-label split, pairs, forward / backward stream slots
 * (with padding), forward / backward arcs actually gathered per frame and utterance */
int ccb_den_info(long *info);

/* scratch sizes for N utterances x T frames on the current device's den graph */
size_t ccb_den_alpha_floats(int N, int T);   /* alpha spill, floats */
size_t ccb_den_aux_bytes(int N, int T);      /* everything else the den passes need */
size_t ccb_ctc_workspace_bytes(int N, int T, int max_label_len);

/* Denominator only: logZ (N,) fp32 device out; grad (strided, pre-zeroed, accumulated with
 * grad_scale); logz_beta may be NULL. */
int ccb_den_forward_backward(const void *logits, int dtype, long sn, long st, int N, int T, int V,
                             const int *len_dev, float *alpha_ws, void *aux_ws,
                             float *grad, long gsn, long gst, float grad_scale,
                             float *logz, float *logz_beta, void *stream);

/* Numerator only: meta_dev = device int32 block [labels(sumL) | label_off(N+1) | label_len(N) | len(N)];
 * grad accumulated with grad_scale (pass e.g. -(1+lamb)/N); logp (N,) fp32 device out. */
int ccb_ctc_forward_backward(const void *logits, int dtype, long sn, long st, int N, int T, int V,
                             const int *labels_dev, const int *label_off_dev, const int *label_len_dev,
                             const int *len_dev, int max_label_len, int blank, void *workspace,
                             float *grad, long gsn, long gst, float grad_scale, float *logp, void *stream);

/* Fused CTC-CRF loss (ctc_crf/__init__.py:58-90 in one call, no host synchronisation) of an (N,T,V) block:
 *   loss[0] = scale * sum_n (logZ_den[n] - (1+lamb) logp_ctc[n])
 *   grad    = scale * (gamma_den - (1+lamb) gamma_ctc)                     (N,T,V) fp32, zeroed here
 * scale = 1/batch for size_average (the caller may split a batch into several calls and sum the losses).
 * Tmax <= T is the number of frames actually walked (max input length of the block); workspaces are sized with
 * ccb_*_floats/bytes(N, Tmax).  parts (optional, may be NULL): 2N floats = [logZ_den | logp_ctc].
 * Everything is enqueued on `stream`. */
int ccb_ctc_crf_loss_fwd(const void *logits, int dtype, int N, int T, int V, int Tmax,
                         const int *labels_dev, const int *label_off_dev, const int *label_len_dev,
                         const int *len_dev, int max_label_len, float lamb, float scale,
                         float *alpha_ws, void *aux_ws, void *ctc_ws,
                         float *grad, float *loss, float *parts, void *stream);

/* Same, taking the RAW encoder outputs z (N,T,V) instead of log-probs (SURVEY 8f-1; replaces the caller's
 * `logits.log_softmax(-1)` + its autograd backward, cat/ctc/train.py:173-174,184-190):
 *   loss as above evaluated on y = log_softmax(z);   grad = d loss / d z = g - softmax(z) * sum_k g_k.
 * No normalised copy of the logits is materialised. */
int ccb_ctc_crf_loss_logits_fwd(const void *logits, int dtype, int N, int T, int V, int Tmax,
                                const int *labels_dev, const int *label_off_dev, const int *label_len_dev,
                                const int *len_dev, int max_label_len, float lamb, float scale,
                                float *alpha_ws, void *aux_ws, void *ctc_ws,
                                float *grad, float *loss, float *parts, void *stream);

/* Checkpointed denominator: the two fused entries above with the alpha memory bounded.  The forward pass keeps alpha on a
 * ring of a few frames plus a copy of every ckpt_k-th frame; the backward pass walks segments of ckpt_k frames from the last
 * to the first, recomputing each from its checkpoint first (one more forward recursion in total).  alpha_ws holds
 * ccb_den_ckpt_alpha_floats(N, Tmax, ckpt_k) floats, about (ceil(Tmax/K) + K + 3) frames of S x PadLanes(N) floats;
 * ckpt_k = 0 is the full spill (ccb_den_alpha_floats).  Same results as the full spill to fp32 rounding.  Costs one more
 * forward recursion: +40 % step time at N=64, T=1500 on an H100 (DESIGN.md "Checkpointed α"). */
size_t ccb_den_ckpt_alpha_floats(int N, int T, int ckpt_k);
int ccb_ctc_crf_loss_ckpt_fwd(const void *logits, int dtype, int N, int T, int V, int Tmax, int ckpt_k,
                              const int *labels_dev, const int *label_off_dev, const int *label_len_dev,
                              const int *len_dev, int max_label_len, float lamb, float scale,
                              float *alpha_ws, void *aux_ws, void *ctc_ws,
                              float *grad, float *loss, float *parts, void *stream);
int ccb_ctc_crf_loss_logits_ckpt_fwd(const void *logits, int dtype, int N, int T, int V, int Tmax, int ckpt_k,
                                     const int *labels_dev, const int *label_off_dev, const int *label_len_dev,
                                     const int *len_dev, int max_label_len, float lamb, float scale,
                                     float *alpha_ws, void *aux_ws, void *ctc_ws,
                                     float *grad, float *loss, float *parts, void *stream);

/* Forward-only CTC-CRF loss, for evaluation without a gradient (CTC_CRF_LOSS under torch.no_grad): the loss and parts of
 * the two fused entries above, from_logits != 0 selecting the raw-logit one, and nothing else.
 *   loss[0] = scale * sum_n (logZ_den[n] - (1+lamb) logp_ctc[n]);   parts (optional, may be NULL): 2N floats [logZ_den | logp_ctc]
 * The den forward pass keeps alpha on a ring of a few frames and sums logZ at each utterance's last frame, so its memory does
 * not grow with Tmax: alpha_ws holds ccb_den_fwd_alpha_floats(N) floats (7 frames of S x PadLanes(N) floats).  There is no
 * backward pass, no numerator cell spill and no (N,T,V) gradient.  aux_ws: ccb_den_aux_bytes(N, Tmax) bytes; num_ws:
 * ccb_num_fwd_only_bytes(N) bytes, the numerator's log-likelihoods.  logp_ctc is bit-identical to the fused entries', logZ_den
 * equal to fp32 rounding.  Everything is enqueued on `stream`. */
size_t ccb_den_fwd_alpha_floats(int N);
size_t ccb_num_fwd_only_bytes(int N);
int ccb_ctc_crf_loss_fwd_only(const void *logits, int dtype, int from_logits, int N, int T, int V, int Tmax,
                              const int *labels_dev, const int *label_off_dev, const int *label_len_dev,
                              const int *len_dev, int max_label_len, float lamb, float scale,
                              float *alpha_ws, void *aux_ws, void *num_ws,
                              float *loss, float *parts, void *stream);

/* CTC-only loss (replaces the numerator-only path ctc_crf/__init__.py:25-56 = WARP_CTC_LOSS) on an (N,T,V) block of
 * log-probs, read in place (no (T,N,V) transpose copy, cf. __init__.py:31):
 *   logp[n] = log p(l_n | x_n)  (N,) device out;   loss[0] = -scale * sum_n logp[n];
 *   grad    = -scale * gamma_ctc, (N,T,V) fp32, every row WRITTEN here (zeros for t >= len and infeasible utterances), so
 *             the caller needs no zero fill (cf. __init__.py:32) and no host round trip for the costs (:35).
 * ctc_ws: ccb_ctc_workspace_bytes(N, Tmax, max_label_len). */
int ccb_ctc_loss_fwd(const void *logits, int dtype, int N, int T, int V, int Tmax,
                     const int *labels_dev, const int *label_off_dev, const int *label_len_dev, const int *len_dev,
                     int max_label_len, int blank, float scale, void *ctc_ws, float *grad, float *loss, float *logp,
                     void *stream);
/* Its forward-only counterpart (WARP_CTC_LOSS under torch.no_grad): logp and loss as above, bit-identical; no workspace and
 * no gradient (one alpha chain per utterance, no cells written). */
int ccb_ctc_loss_fwd_only(const void *logits, int dtype, int N, int T, int V, int Tmax,
                          const int *labels_dev, const int *label_off_dev, const int *label_len_dev, const int *len_dev,
                          int max_label_len, int blank, float scale, float *loss, float *logp, void *stream);

/* Per-utterance costs (reduction 'none') and zero_infinity.  The loss entries above with two more arguments:
 *   costs    (optional, may be NULL): N floats out, cost[n] = logZ_den[n] - (1+lamb) logp_ctc[n] (CTC-CRF) or -logp[n] (CTC),
 *            unscaled; loss[0] = scale * sum_n cost[n] as before.  A batch split into several calls passes costs + n0.
 *   zero_inf (0 / 1): an utterance whose cost is not finite (+-inf or NaN: an infeasible label sequence, an utterance that
 *            cannot reach a final state of the den graph, a length of 0) gets cost 0 in `costs` and in the sum, and zero
 *            gradient rows -- den part included -- in every row t < len.  The mask is applied on the device, by the kernels
 *            that already read both halves of the loss; nothing synchronises the host.
 * With costs = NULL and zero_inf = 0 each is exactly the entry it extends.
 * ccb_ctc_crf_loss_costs: ccb_ctc_crf_loss_fwd / _logits_fwd / _ckpt_fwd / _logits_ckpt_fwd, selected by from_logits != 0 and
 * ckpt_k > 0 (ckpt_k = 0: the full alpha spill). */
int ccb_ctc_crf_loss_costs(const void *logits, int dtype, int from_logits, int N, int T, int V, int Tmax, int ckpt_k,
                           const int *labels_dev, const int *label_off_dev, const int *label_len_dev,
                           const int *len_dev, int max_label_len, float lamb, float scale,
                           float *alpha_ws, void *aux_ws, void *ctc_ws,
                           float *grad, float *loss, float *parts, float *costs, int zero_inf, void *stream);
/* ccb_ctc_crf_loss_fwd_only with costs and zero_inf (no gradient, so zero_inf masks the costs and the sum only). */
int ccb_ctc_crf_loss_costs_fwd_only(const void *logits, int dtype, int from_logits, int N, int T, int V, int Tmax,
                                    const int *labels_dev, const int *label_off_dev, const int *label_len_dev,
                                    const int *len_dev, int max_label_len, float lamb, float scale,
                                    float *alpha_ws, void *aux_ws, void *num_ws,
                                    float *loss, float *parts, float *costs, int zero_inf, void *stream);
/* ccb_ctc_loss_fwd with costs and zero_inf; grad = NULL is ccb_ctc_loss_fwd_only (ctc_ws is then not used, may be NULL). */
int ccb_ctc_loss_costs(const void *logits, int dtype, int N, int T, int V, int Tmax,
                       const int *labels_dev, const int *label_off_dev, const int *label_len_dev, const int *len_dev,
                       int max_label_len, int blank, float scale, void *ctc_ws, float *grad, float *loss, float *logp,
                       float *costs, int zero_inf, void *stream);
/* Backward of a loss with per-utterance costs: out[n][t][:] = w[n] * grad[n][t][:] for t < len[n], zeros beyond (grad is
 * not read there), in one pass.  grad: (N,T,V) fp32, the unscaled gradient of the entries above (scale = 1); w: (N,) fp32,
 * the gradient of the caller's objective with respect to each cost; out: (N,T,V) in the CCB_DTYPE_* code out_dtype (fp32,
 * bf16 or fp16, rounded to nearest), not aliasing grad. */
int ccb_grad_rows_scale(const float *grad, const float *w, const int *len_dev, int N, int T, int V, void *out, int out_dtype,
                        void *stream);

/* Several label sequences per utterance (sampled sequences, N-best lists, alternative pronunciations), with the den passes run
 * once per utterance.  M sequences, grouped by utterance (the sequences of utterance n are seq_off[n] .. seq_off[n+1]-1):
 *   labels_dev / label_off_dev / label_len_dev describe the M sequences in that order (label_off: M entries);
 *   len_dev      (N,) frames per utterance;
 *   seq_row_dev  (M,) the logits row, in [0, N), sequence m is scored against;
 *   seq_pos_dev  (M,) the index of sequence m in the caller's order: costs[seq_pos[m]] (and w[seq_pos[m]]) belong to it;
 *   seq_off_dev  (N+1,) offsets of each utterance's sequences; seq_off[0] is the first sequence of this call.
 *   cost[m] = logZ_den[seq_row[m]] - (1+lamb) logp_ctc[m] (CTC-CRF) or -logp[m] (CTC); loss[0] = scale * sum_m cost[m];
 *   grad[n] = sum_{m of n} w_m (gamma_den[n] - (1+lamb) gamma_ctc[m]), w_m = scale (CTC-CRF; CTC: -scale gamma_ctc[m] alone).
 * The den occupancies are computed once per utterance and scaled by W_n = sum of w_m over its unmasked sequences; an utterance
 * without an unmasked sequence (or without any) gets zero rows.  zero_inf masks per sequence.  logp_ctc[m] is bit-identical to
 * a single-sequence call on row seq_row[m].  ctc_ws: ccb_ctc_workspace_bytes(M, Tmax, max_label_len); alpha_ws / aux_ws as
 * for N utterances.  M = 0 is allowed (zero rows, loss 0).
 * defer_num != 0 (reduction 'none' with a gradient): grad receives the UNSCALED den occupancies only (CTC: grad is not used),
 * and the numerator's cells stay in ctc_ws for ccb_seqs_grad, which the caller runs later with its per-sequence weights. */
int ccb_ctc_crf_loss_seqs(const void *logits, int dtype, int from_logits, int N, int T, int V, int Tmax, int ckpt_k,
                          const int *labels_dev, const int *label_off_dev, const int *label_len_dev, const int *len_dev,
                          int M, const int *seq_row_dev, const int *seq_pos_dev, const int *seq_off_dev, int max_label_len,
                          float lamb, float scale, float *alpha_ws, void *aux_ws, void *ctc_ws, float *grad, float *loss,
                          float *costs, int zero_inf, int defer_num, void *stream);
/* Its forward-only counterpart (ccb_ctc_crf_loss_fwd_only's passes); num_ws: ccb_num_fwd_only_bytes(M). */
int ccb_ctc_crf_loss_seqs_fwd_only(const void *logits, int dtype, int from_logits, int N, int T, int V, int Tmax,
                                   const int *labels_dev, const int *label_off_dev, const int *label_len_dev,
                                   const int *len_dev, int M, const int *seq_row_dev, const int *seq_pos_dev,
                                   int max_label_len, float lamb, float scale, float *alpha_ws, void *aux_ws, void *num_ws,
                                   float *loss, float *costs, int zero_inf, void *stream);
/* CTC-only loss over M sequences: logp (M,) out in the grouped order.  ctc_ws = NULL: forward only (no cells, grad unused);
 * otherwise every row of the (N,T,V) grad is written (unless defer_num). */
int ccb_ctc_loss_seqs(const void *logits, int dtype, int N, int T, int V, int Tmax,
                      const int *labels_dev, const int *label_off_dev, const int *label_len_dev, const int *len_dev,
                      int M, const int *seq_row_dev, const int *seq_pos_dev, const int *seq_off_dev, int max_label_len,
                      int blank, float scale, void *ctc_ws, float *grad, float *loss, float *logp, float *costs,
                      int zero_inf, int defer_num, void *stream);
/* The deferred gradient of a defer_num call, with per-sequence weights w (M,) in the caller's order:
 *   out[n] = W_n den[n] + num_coef * sum_{m of n} w[seq_pos[m]] gamma_ctc[m],  W_n = sum of w over the unmasked sequences of n
 * written to every row of the (N,T,V) fp32 `out` (zeros for t >= len); den = NULL for the CTC-only loss.  from_logits != 0
 * chains it through log_softmax as the fused entry does.  aux_ws / ctc_ws: the forward call's, untouched since; out may not
 * alias den.  num_coef: -(1+lamb) for CTC-CRF, -1 for CTC. */
int ccb_seqs_grad(const void *logits, int dtype, int from_logits, int N, int T, int V, int Tmax,
                  const int *labels_dev, const int *label_off_dev, const int *label_len_dev, const int *len_dev,
                  int M, const int *seq_pos_dev, const int *seq_off_dev, int max_label_len, int blank, float num_coef,
                  const float *w, const float *den, void *aux_ws, void *ctc_ws, int zero_inf, float *out, void *stream);
/* ccb_ctc_align over M sequences: align (M,T) and score (M,) in the caller's order (row seq_pos[m]); workspace:
 * ccb_ctc_align_workspace_bytes(M, T, max_label_len). */
int ccb_ctc_align_seqs(const void *logits, int dtype, long sn, long st, int N, int T, int V,
                       const int *labels_dev, const int *label_off_dev, const int *label_len_dev, const int *len_dev,
                       int M, const int *seq_row_dev, const int *seq_pos_dev, int max_label_len, int blank, void *workspace,
                       int *align, float *score, void *stream);

/* Best-path (Viterbi) alignment over the numerator lattice -- the forced alignment that comes with the CTC numerator
 * (SURVEY.md 8f-4).  align: (N,T) int32 device out, the token emitted at every frame t < len (blank included), -1 beyond
 * the length and for infeasible utterances; score (optional, may be NULL): (N,) log-probability of the best path.
 * workspace: ccb_ctc_align_workspace_bytes(N, T, max_label_len) bytes. */
size_t ccb_ctc_align_workspace_bytes(int N, int T, int max_label_len);
int ccb_ctc_align(const void *logits, int dtype, long sn, long st, int N, int T, int V,
                  const int *labels_dev, const int *label_off_dev, const int *label_len_dev, const int *len_dev,
                  int max_label_len, int blank, void *workspace, int *align, float *score, void *stream);

/* Exact samples from the CTC-CRF posterior p(path | x) over the den graph loaded by Init (forward filtering, backward
 * sampling): K paths per utterance, each drawn with probability w(path) prod_t exp(y[t][lab]) final / Z.  The den forward
 * pass runs once per utterance; then one warp per (utterance, sample) walks back from a final state drawn with probability
 * ~ alpha_len(q) final(q), drawing at every frame a predecessor p with probability ~ alpha_{t-1}(p) w_pq.
 *   logits   (N,T,V) log-probs or raw logits in the CCB_DTYPE_* code dtype (the same distribution: the per-frame log-softmax
 *            shift cancels); only frames t < len are read.
 *   Tmax     the longest length (<= T); ckpt_k 0: the full alpha spill, > 0: checkpointed alpha (ccb_ctc_crf_loss_ckpt_fwd),
 *            each segment recomputed and walked, the last one first.  alpha_ws / aux_ws as for the loss entries.
 *   seed     64-bit Philox4x32-10 key; the uniform that picks the state of frame t of sample k of utterance n is counter
 *            (t, k, n_base + n, 0), so an utterance's samples do not depend on the rest of the batch.
 *   sample_ws  ccb_crf_sample_ws_bytes(N, K, Tmax) bytes.
 *   tokens (N,K,T) int32 out: the CTC collapse of each path (repeats merged, blank 0 dropped), -1 after the last token;
 *   lengths (N,K) int32 out: token count; align (N,K,T) int32 out: the label of every frame t < len (blank included), -1
 *   beyond; path_logp (N,K) fp32 out: log p(path | x), accumulated in fp64.  An utterance with no path of finite score (length
 *   0, -inf frames, no final state reachable) gets length -1, rows of -1 and -inf.  Everything is enqueued on `stream`; the
 *   first call on a device uploads the graph's in-arc table (about 8 bytes per arc) synchronously. */
size_t ccb_crf_sample_ws_bytes(int N, int K, int T);
int ccb_crf_sample(const void *logits, int dtype, int N, int T, int V, int Tmax, int ckpt_k, const int *len_dev, int K,
                   unsigned long long seed, int n_base, float *alpha_ws, void *aux_ws, void *sample_ws, int *tokens,
                   int *lengths, int *align, float *path_logp, void *stream);

/* CTC prefix beam search: the `beam` best label sequences of every utterance, one CTA per utterance, one launch.
 *   crf 0: plain CTC -- a path is any frame-label sequence, scored sum_t y[t][lab_t];
 *   crf 1: over the split den graph loaded by Init -- a path is a state sequence from the start state, scored
 *          sum log w(arcs) + sum_t y[t][lab(q_t)] + log final(q_len): for a T-compose-LM graph, a label sequence's total is
 *          log p_LM(l) + log p_ctc(l|x).  The graph must pass the CTC-shape check (ccb_plan_ctc_shape), run once per graph
 *          and device at the first crf=1 call, which also uploads the out-arc table (about 12 bytes per arc) synchronously.
 * A hypothesis's score is the log-sum of the scores of its paths the beam kept (fp64 inside): a lower bound on the exact
 * log mass of the sequence, equal to it when nothing was pruned.  Raw logits give the same hypotheses as their log-softmax,
 * with every score shifted by sum_t logsumexp(y[t]).
 *   logits   (N,T,V) contiguous in the CCB_DTYPE_* code dtype; only frames t < len are read.  V <= 8192.
 *   beam     1 .. 128; cutoff_top_n 1 .. V: the tokens of a frame are its cutoff_top_n largest entries (ties: lower id),
 *            plus blank and each hypothesis's own last token.  Ties between candidates break on (parent rank, token).
 *   workspace  ccb_ctc_beam_search_ws_bytes(N, T, beam) bytes; nothing needs to be initialised.
 *   tokens (N,beam,T) int32 out, -1 padded; lengths (N,beam) int32 out; timesteps (N,beam,T) int32 out: the frame at
 *   which the trie node of each token was created, -1 padded; scores (N,beam) fp32 out, best first.  Rows beyond the
 *   hypotheses of finite score get length -1, tokens and timesteps -1 and score -inf.  len = 0 gives the empty sequence,
 *   scored 0 (crf 0) or log final(start) (crf 1). */
size_t ccb_ctc_beam_search_ws_bytes(int N, int T, int beam);
int ccb_ctc_beam_search(const void *logits, int dtype, int N, int T, int V, const int *len_dev, int beam, int cutoff_top_n,
                        int crf, void *workspace, int *tokens, int *lengths, int *timesteps, float *scores, void *stream);

/* Token-level shallow fusion of a back-off n-gram LM into the plain (crf 0) prefix beam search.  A hypothesis l = l_1..l_k
 * scores  A(l) + alpha sum_{i=1..k+1} ln P(w_i | w_{i-n+1} .. w_{i-1}) + beta k,  where A(l) is ccb_ctc_beam_search's score,
 * w_i = labels[l_i] (w_0 = <s> when the LM lists it, w_{k+1} = </s>) and P is ARPA back-off (log10 values, fp32 as parsed,
 * turned into natural log in fp64).  An extension p -> p+c adds alpha ln P(c | p) + beta to the candidate's rank during the
 * search; the </s> term is added after the last frame and the hypotheses re-ranked.  alpha = 0 does not consult the LM.
 *   ccb_ngram_create: parse the ARPA text at `path` for the token labels labels[0..V) (labels[0], the blank, is never scored;
 *     a label the LM does not list, or an empty one, scores as <unk>; <s> or </s> as a label is an error).  Host only, no CUDA.
 *     NULL on failure, with ccb_last_error naming the line.  KenLM binaries and compressed files are not read.
 *   ccb_ngram_destroy: frees the host tables and the device copies; it calls cudaFree, which waits for the device.
 *   ccb_ngram_info: info[0..7] = order, states, arcs, <unk> substituted (0/1), words, V, state after <s>, word id of </s>;
 *     info[8..17] = n-gram counts of orders 1..10 as \data\ declares them (0 past the order).
 *   ccb_ngram_copy (tests): which 0 tok2word[V] i32, 1 root_p[W] f32, 2 root_dst[W] i32, 3 arc_off[S+1] i32, 4 arc_word[A]
 *     i32, 5 arc_p[A] f32 (NaN: a prefix inserted by the closure, whose value is the back-off value), 6 arc_dst[A] i32,
 *     7 bow[S] f32, 8 back[S] i32 (ngram.h NGramHost).
 *   ccb_ctc_beam_search_lm: ccb_ctc_beam_search with the LM fused in; lm = NULL is ccb_ctc_beam_search.  crf must be 0, alpha
 *     finite and >= 0, beta finite, V the LM's label count.  The first search with an LM on a device uploads its tables
 *     (about 12 bytes per arc) synchronously; the workspace is the same. */
void *ccb_ngram_create(const char *path, const char *const *labels, int V);
void ccb_ngram_destroy(void *lm);
int ccb_ngram_info(void *lm, long *info);
int ccb_ngram_copy(void *lm, int which, void *dst, size_t dst_bytes);
int ccb_ctc_beam_search_lm(const void *logits, int dtype, int N, int T, int V, const int *len_dev, int beam, int cutoff_top_n,
                           int crf, void *workspace, int *tokens, int *lengths, int *timesteps, float *scores, const void *lm,
                           double alpha, double beta, void *stream);

/* 1-best word decoding through a TLG decoding graph: a frame-synchronous Viterbi beam search on the GPU, the 1-best step of
 * Kaldi's latgen-faster + lattice-best-path without the lattice (DESIGN.md §7 "TLG decoding").  The graph is an OpenFst
 * vector/standard file in CAT's conventions: ilabel = token + 1 (blank = token 0), ilabel 0 = epsilon, olabel = word id
 * (0 = no word), tropical weights.  With acs = acwt / lmwt and wps = wip / lmwt (fp32), the search cost of an emitting arc
 * from a token of cost c is ((c + w) + (-acs * y[t][token])) + (word ? wps : 0), of an epsilon arc (c + w) + (word ? wps : 0),
 * each operation rounded in fp32.  Each frame keeps the tokens within best + beam (best: the cheapest emitting candidate),
 * recombines per state on the smallest (cost, arc position in the file), runs the epsilon closure by increasing epsilon
 * level, and keeps the max_active cheapest by (cost, state).  The result is the kept token with the smallest
 * (cost + final, state), or without a final state among them the smallest (cost, state) with reached_final = 0.
 *   ccb_wfst_create: read the file and derive the arc layout, the epsilon levels and the sizes below.  Host only, no CUDA.
 *     NULL on failure, with ccb_last_error saying what is wrong: an epsilon cycle (naming a state on it), a const FST, an
 *     embedded symbol table or an aligned file (each with the conversion to run).  Several graphs may coexist, and none
 *     depends on the den graph of Init.
 *   ccb_wfst_destroy: frees the host tables and the device copies; it calls cudaFree, which waits for the device.
 *   ccb_wfst_info: info[0..7] = states, arcs, start, L (the longest epsilon path), E (the most states one state reaches
 *     through epsilon arcs), the largest emitting out-degree, the largest ilabel, epsilon arcs.
 *   ccb_wfst_copy (tests): which 0 arc_off[S+1], 1 eps_off[S] (each state's arcs: emitting ones, in file order, up to
 *     eps_off, then epsilon ones), 2 dst[A], 3 token[A] (-1: epsilon), 4 olabel[A], 5 weight[A] f32, 6 file position[A],
 *     7 final[S] f32 (+inf: not final), 8 epsilon level[S]; i32 unless stated.
 *   ccb_wfst_decode_ws_bytes: the workspace of N utterances of T frames; 0 for bad arguments.
 *   ccb_wfst_decode: logits (N,T,V) log-probs or raw logits in dtype, frames t >= len_dev[n] never read; max_active in
 *     [1, 2^20], beam > 0 (inf allowed), acwt finite >= 0, lmwt finite > 0, wip finite, V <= 8192 and at least the graph's
 *     largest ilabel.  Outputs, written on `stream` without a host synchronisation, in one launch:
 *       words (N, Wcap) i32 padded with -1, Wcap = (T+1)(1+L); num_words (N) i32; align (N,T) i32: the token of each frame's
 *       emitting arc, -1 for t >= len; ac_logp (N) = sum_t y[t][align[t]] and graph_cost (N) = the path's weights plus its
 *       final cost, both summed in fp64; cost (N) = lmwt graph_cost - acwt ac_logp + wip num_words (lattice-best-path's
 *       objective); reached_final (N) i32.  An utterance whose candidates all cost +inf gets num_words -1, rows of -1,
 *       ac_logp -inf and graph_cost and cost +inf.  The first search with a graph on a device uploads its tables (about 36
 *       bytes per arc) synchronously. */
void *ccb_wfst_create(const char *path);
void ccb_wfst_destroy(void *graph);
int ccb_wfst_info(void *graph, long *info);
int ccb_wfst_copy(void *graph, int which, void *dst, size_t dst_bytes);
size_t ccb_wfst_decode_ws_bytes(void *graph, int N, int T, int max_active);
int ccb_wfst_decode(const void *logits, int dtype, int N, int T, int V, const int *len_dev, void *graph, float acwt,
                    float lmwt, float wip, float beam, int max_active, void *workspace, int *words, int *num_words,
                    int *align, float *ac_logp, float *graph_cost, float *cost, int *reached_final, void *stream);

/* RNN-T loss (DESIGN.md §7 "RNN-T loss"), the textbook transducer loss over a joint tensor x of log-probs (from_logits = 0)
 * or raw joiner outputs (from_logits = 1: the log-softmax is taken inside, no normalised copy is written).  Utterance n has
 * T_n = lx[n] >= 1 frames and U_n = ly[n] >= 0 labels y_1..y_U; with lp(t,u,k) the log-prob of token k at row (t,u),
 *   alpha(0,0) = 0,  alpha(t,u) = logaddexp(alpha(t-1,u) + lp(t-1,u,blank), alpha(t,u-1) + lp(t,u-1,y_u)),
 *   cost[n] = -(alpha(T-1,U) + lp(T-1,U,blank)).
 * Layouts (x is read in place in the CCB_DTYPE_* code dtype; all arithmetic in fp32, the lattice cells in fp64):
 *   compact != 0: x (rows, V), utterance n at rows off_n + t (U_n+1) + u, off_n = sum_{m<n} T_m (U_m+1), computed on the
 *     device in int64; labels (n_labels,) the label sequences concatenated.  Rows behind the last utterance are not read.
 *   compact == 0: x (N, Tmax, Umax+1, V) = rows of N Tmax (Umax+1); labels (N, Umax) = n_labels of N Umax.  Rows outside
 *     t < T_n, u <= U_n are never read.
 * An utterance whose lengths overrun the tensor or the labels (or T_n < 1, U_n < 0, or T_n > Tmax, U_n > Umax when padded), or
 * with a label outside [0, V) or equal to blank, gets cost NaN and zero gradient rows; nothing outside the tensors is read.
 * No atomics: two identical calls give identical bits.
 *   ccb_rnnt_workspace_bytes: the workspace of a call, about 28 bytes per row (lp of blank and label, the row's logsumexp,
 *     alpha and beta in fp64) plus 56 bytes per utterance.  Nothing needs to be initialised.
 *   ccb_rnnt_forward: costs (N,) fp32 out, from alpha.  want_beta != 0 also runs beta (concurrently with alpha, one CTA per
 *     utterance and direction), which ccb_rnnt_backward needs; costs_beta (N,) (optional, may be NULL) then gets
 *     -beta(0,0), the same cost from the other direction.  Lengths and labels are device pointers; no host synchronisation.
 *   ccb_rnnt_backward: after a want_beta forward on the same workspace (untouched since) and the same x, labels and
 *     lengths: grad (the shape of x, in dtype) = w[n] d cost[n] / d x for every row of utterance n, and zeros in every other
 *     row (not read), in one pass.  With pb / pl the posteriors of the blank / label transition out of row (t,u):
 *     log-prob input: -pb at blank, -pl at y_{u+1}, 0 elsewhere; raw logits: softmax(x) (pb + pl) minus the same two terms.
 *     w (N,) fp32 device: the caller's weight of each cost (1/N for a batch mean).  x is read only when from_logits. */
size_t ccb_rnnt_workspace_bytes(int N, long rows);
int ccb_rnnt_forward(const void *x, int dtype, int from_logits, int compact, int N, long rows, int V, int Tmax, int Umax,
                     const int *labels_dev, long n_labels, const int *lx_dev, const int *ly_dev, int blank, int want_beta,
                     void *workspace, float *costs, float *costs_beta, void *stream);
int ccb_rnnt_backward(const void *x, int dtype, int from_logits, int N, long rows, int V, const int *labels_dev, int blank,
                      void *workspace, const float *w, void *grad, void *stream);

/* RNN-T loss of CAT's LogAdd joiner, from the encoder output f (N, Tmax, V) and the predictor output g (N, Umax+1, V)
 * without the joint tensor: with z(t,u,k) = f[n,t,k] + g[n,u,k] (fp32 sum of the values as given) and
 * Z(t,u) = logsumexp_k z(t,u,k), the lattice of ccb_rnnt_forward has lp(t,u,k) = z(t,u,k) - Z(t,u).  f and g share the
 * CCB_DTYPE_* code dtype and are read in place; labels (N, Umax), lx, ly (N,) int32 device.  Rows t >= T_n of f and u > U_n of
 * g are never read.  An utterance with T_n < 1, U_n < 0, T_n > Tmax, U_n > Umax, or a label outside [0, V) or equal to
 * blank, gets cost NaN and zero gradient rows.  Z is mf_t + mg_u + log S(t,u) with the row maxima mf, mg and
 * S = sum_k exp(f[t,k] - mf_t) exp(g[u,k] - mg_u) from an fp32 GEMM; a cell with S < 2^-64 takes Z from an exact logsumexp
 * over f[t] + g[u] instead.  No atomics: two identical calls give identical bits.  N <= 65535.
 *   ccb_rnnt_simple_workspace_bytes: the workspace of a call, sized from the shapes alone: 44 bytes per cell of the padded
 *     lattice, N Tmax (Umax+1) cells (lp of blank and label, Z, alpha and beta in fp64 as ccb_rnnt_forward; S, the cell
 *     weight and the weighted blank and label posteriors in fp32), 8 bytes per row of f and of g (row maximum, flag) and
 *     56 bytes per utterance, each block aligned to 256 bytes.  Nothing needs to be initialised.
 *   ccb_rnnt_simple_forward: costs (N,) fp32 out.  want_beta != 0 also runs beta, which ccb_rnnt_simple_backward needs.
 *   ccb_rnnt_simple_backward: after a want_beta forward on the same workspace (untouched since) and the same f, g, labels
 *     and lengths: grad_f (the shape of f) and grad_g (the shape of g), in dtype, = w[n] d cost[n] / d f and d g, with
 *     zeros in every row outside the utterances (not read).  The workspace may serve several backward calls. */
size_t ccb_rnnt_simple_workspace_bytes(int N, int Tmax, int Umax);
int ccb_rnnt_simple_forward(const void *f, const void *g, int dtype, int N, int Tmax, int Umax, int V, const int *labels_dev,
                            const int *lx_dev, const int *ly_dev, int blank, int want_beta, void *workspace, float *costs,
                            void *stream);
int ccb_rnnt_simple_backward(const void *f, const void *g, int dtype, int N, int Tmax, int Umax, int V, const int *labels_dev,
                             int blank, void *workspace, const float *w, void *grad_f, void *grad_g, void *stream);

/* CTC-T loss (DESIGN.md §7 "CTC-T loss"), the loss of CAT's `topo: ctct` transducers: every frame emits exactly one symbol,
 * as in CTC, and reads the row of the labels emitted so far, as in RNN-T.  Over the states (u, b) (u labels emitted, the
 * last emission blank or none yet) and (u, l) (u >= 1, the last emission y_u), with lp(t,u,k) the log-prob of token k at row
 * (t,u), alpha_0(0,b) = 0 and every other alpha_0 = -inf, and logaddexp written (+):
 *   alpha_{t+1}(u,b) = [alpha_t(u,b) (+) alpha_t(u,l)] + lp(t,u,blank)
 *   alpha_{t+1}(u,l) = [alpha_t(u,l) + lp(t,u,y_u)] (+) [alpha_t(u-1,b) + lp(t,u-1,y_u)]
 *                      (+) [alpha_t(u-1,l) + lp(t,u-1,y_u)]   (only if u = 1 or y_u != y_{u-1})
 *   cost[n] = -(alpha_T(U,b) (+) alpha_T(U,l)).
 * Each entry takes the arguments of its RNN-T counterpart and keeps its conventions: layouts, fp64 cells, NaN cost and zero
 * gradient rows for a bad utterance, no atomics, no host synchronisation.  An infeasible utterance (T_n < U_n + the number of
 * adjacent repeats in its labels) gets cost +inf and zero gradient, never NaN.
 *   ccb_ctct_workspace_bytes: about 48 bytes per row (alpha and beta as two fp64 cells each; lp of blank, of y_{u+1} and of
 *     y_u and the row's logsumexp in fp32) plus 56 bytes per utterance.  Nothing needs to be initialised.
 *   ccb_ctct_forward: as ccb_rnnt_forward; costs_beta gets -beta_0(0,b).
 *   ccb_ctct_backward: as ccb_rnnt_backward, with pb, pr and pl the posteriors of the blank, the repeat of y_u and the new
 *     label y_{u+1} read at row (t,u): log-prob input: -pb at blank, -pr at y_u, -pl at y_{u+1} (added where y_u = y_{u+1});
 *     raw logits: softmax(x) (pb + pr + pl) minus the same terms. */
size_t ccb_ctct_workspace_bytes(int N, long rows);
int ccb_ctct_forward(const void *x, int dtype, int from_logits, int compact, int N, long rows, int V, int Tmax, int Umax,
                     const int *labels_dev, long n_labels, const int *lx_dev, const int *ly_dev, int blank, int want_beta,
                     void *workspace, float *costs, float *costs_beta, void *stream);
int ccb_ctct_backward(const void *x, int dtype, int from_logits, int N, long rows, int V, const int *labels_dev, int blank,
                      void *workspace, const float *w, void *grad, void *stream);

/* CTC-T loss of CAT's LogAdd joiner, lp(t,u,k) = f[n,t,k] + g[n,u,k] - Z(t,u) as for ccb_rnnt_simple_forward, with the
 * lattice of ccb_ctct_forward.  Arguments and conventions as the ccb_rnnt_simple_* entries.
 *   ccb_ctct_simple_workspace_bytes: the layout of ccb_rnnt_simple_workspace_bytes with the CTC-T lattice (two fp64 cells
 *     per direction and lp of y_u per cell) and one more fp32 per cell (the repeat posterior): 68 bytes per cell of the padded
 *     lattice, 8 bytes per row of f and of g and 56 bytes per utterance, each block aligned to 256 bytes. */
size_t ccb_ctct_simple_workspace_bytes(int N, int Tmax, int Umax);
int ccb_ctct_simple_forward(const void *f, const void *g, int dtype, int N, int Tmax, int Umax, int V, const int *labels_dev,
                            const int *lx_dev, const int *ly_dev, int blank, int want_beta, void *workspace, float *costs,
                            void *stream);
int ccb_ctct_simple_backward(const void *f, const void *g, int dtype, int N, int Tmax, int Umax, int V, const int *labels_dev,
                             int blank, void *workspace, const float *w, void *grad_f, void *grad_g, void *stream);

/* The compact joiner's broadcast sum (CAT's gather.sum): for N utterances with la[n] rows of a and lb[n] rows of b, laid out
 * one utterance after the other in each (offsets ta_n, ub_n and off_n = sum_{m<n} la_m lb_m computed on the device),
 *   out[off_n + t lb_n + u][h] = a[ta_n + t][h] + b[ub_n + u][h]   (fp32 sum, rounded to dtype),
 * a (sum la, H), b (sum lb, H), out (rows_out = sum la lb, H), all in the CCB_DTYPE_* code dtype; la / lb (N,) int32 device,
 * >= 0 and consistent with the row counts (the caller checks; the kernels trust them).  The backward writes
 * grad_a[ta_n + t] = sum_u grad_out[off_n + t lb_n + u] and grad_b[ub_n + u] = sum_t grad_out[...], each accumulated in fp32
 * in a fixed order, without atomics.  workspace: ccb_gather_ws_bytes(N) bytes. */
size_t ccb_gather_ws_bytes(int N);
int ccb_gather_sum(const void *a, const void *b, int dtype, int N, long rows_out, int H, const int *la_dev, const int *lb_dev,
                   void *workspace, void *out, void *stream);
int ccb_gather_sum_backward(const void *grad_out, int dtype, int N, long rows_a, long rows_b, int H, const int *la_dev,
                            const int *lb_dev, void *workspace, void *grad_a, void *grad_b, void *stream);

/* Transducer (RNN-T, monotonic) beam search, one launch per frame; the caller runs the networks between launches.  Each
 * utterance keeps a beam of `beam` slots (1 .. 128): per slot, parent / token / node int32 and score fp64, all (N, beam)
 * device arrays.  Live slots are a prefix of the beam (score > -inf); the empty prefix is trie node 0.
 *   ccb_rnnt_beam_init: the beam [empty prefix, score 0] and an empty trie.
 *   ccb_rnnt_beam_step (frame t; utterances with t >= len_dev[n] keep their beam, each slot its own parent, token -1):
 *     rows (N*beam, V) in the CCB_DTYPE_* code dtype, row n*beam + q for slot q of utterance n (rows of dead slots are not
 *     read).  mode 0: log-probs; 1: raw joiner logits, normalised by the row's logsumexp; 2: the LogAdd joiner's g rows,
 *     z = f[n, t] + g in fp32 with enc = f (N, Tmax, V) of the same dtype, normalised likewise.  Candidate (r, k) has
 *     value score_r + lp_r[k] (fp64); the min(beam, live * V) best, by value desc then r * V + k asc, -inf dropped, are
 *     merged in increasing r * V + k by target prefix (blank: the slot's own prefix, else prefix + k), logaddexp in fp64.
 *     Each slot of the new beam (order of first appearance) gets its parent slot, token (-1 for blank), trie node and
 *     score; dead slots parent = itself, token -1, node -1, score -inf.  V <= 2^24, blank in [0, V).
 *   ccb_rnnt_beam_finish: the beam ranked by score (stable), the first nbest (1 .. beam) rows written: tokens
 *     (N, nbest, Tmax) int32 -1 padded, lengths (N, nbest) int32 (-1 past the hypotheses found), scores (N, nbest) fp32.
 * workspace: ccb_rnnt_beam_ws_bytes(N, Tmax, beam) bytes (0 for beam outside [1, 128]): per utterance the trie (at most
 * 1 + beam * Tmax nodes) and its hash table; ccb_rnnt_beam_init initialises it. */
size_t ccb_rnnt_beam_ws_bytes(int N, int Tmax, int beam);
int ccb_rnnt_beam_init(int N, int Tmax, int beam, void *workspace, int *parent, int *token, int *node, double *score,
                       void *stream);
int ccb_rnnt_beam_step(const void *rows, const void *enc, int dtype, int mode, int N, int Tmax, int beam, int V, int t,
                       const int *len_dev, int blank, void *workspace, int *parent, int *token, int *node, double *score,
                       void *stream);
int ccb_rnnt_beam_finish(int N, int Tmax, int beam, int nbest, const void *workspace, const int *node, const double *score,
                         int *tokens, int *lengths, float *scores, void *stream);

/* The transducer beam search step with an external LM and / or an internal-LM (ILM) estimate fused in, as CAT's RNNTDecoder
 * does with --alpha / --beta / --ilm-weight (DESIGN.md §7 "RNN-T beam search with LM fusion").  Arguments and slot arrays as
 * ccb_rnnt_beam_step, plus lm_part (N, beam) fp64: each slot's LM part, read for the current beam and written for the next
 * (ccb_rnnt_beam_init does not touch it: zero it for the first frame).  lm_rows (N*beam, V) are the slots' external-LM
 * log-probs, ilm_rows (N*beam, V) their ILM logits, each in its own CCB_DTYPE_* code dtype; a null block turns its term off,
 * and both null is an error.  alpha, beta, ilm_weight: finite, any sign.  Candidate (r, k) ranks by
 *   ((score_r + lp_r[k]) + lm_part_r) + [k != blank] term_r[k],
 *   term_r[k] = (beta + alpha LM_r[k]) + ilm_weight (I_r[k] - logsumexp_{j != blank} I_r[j])   (the absent term dropped),
 * fp64, I_r[k] - lse in fp32; a -inf LM or ILM entry makes the candidate -inf.  Selection and merge as ccb_rnnt_beam_step,
 * except that a new slot's score is the logaddexp of its candidates' acoustic parts score_r + lp_r[k] alone and its LM part
 * is its first candidate's: lm_part_r for blank, lm_part_r + term_r[k] for an extension.  The hypothesis score is
 * score + lm_part: add it into score before ccb_rnnt_beam_finish.  Dead slots get lm_part 0. */
int ccb_rnnt_beam_step_fused(const void *rows, const void *enc, int dtype, int mode, int N, int Tmax, int beam, int V, int t,
                             const int *len_dev, int blank, void *workspace, int *parent, int *token, int *node,
                             double *score, const void *lm_rows, int lm_dtype, double alpha, double beta,
                             const void *ilm_rows, int ilm_dtype, double ilm_weight, double *lm_part, void *stream);
/* A token n-gram LM's (ccb_ngram_create) rows for ccb_rnnt_beam_step_fused.  For every slot q of N*beam: its LM state is
 * state_in[n*beam + parent[q]] advanced by token[q] when token[q] >= 0 (the back-off walk's destination rule), or, with
 * parent null (token and state_in then unused), the state after </s> from the root: the start of every hypothesis.  It is
 * written to state_out[q] (int32, a different array from state_in), and rows[q] (V fp32) gets ln P(label k | state) for
 * every k, the fp64 log10 value times ln 10 rounded once; a label without an LM word (label 0) gets 0.  The LM must have
 * been loaded for V labels and have at most 25600 words. */
int ccb_ngram_slot_rows(const void *lm, int N, int beam, int V, const int *parent, const int *token, const int *state_in,
                        int *state_out, float *rows, void *stream);
/* Sentence scores under a token n-gram LM (ccb_ngram_create), as CAT's NGram.score computes them (DESIGN.md §7 "N-gram
 * sentence scoring"), one launch.  Row b of R: ids + b*ids_stride holds its tokens (U columns, contiguous), last +
 * b*last_stride its last target (CAT's targets[b, -1]), lens[b] its length L (lens null: every L = U); each array is int32,
 * or int64 where its *_i64 flag is 1, on the device, read in place, and only ids[b][0 .. L) is read.  out[b] (fp32) =
 * ln 10 * sum_{i=0..L} log10 P(w_i | w_max(0,i-n+1) .. w_i-1) by ARPA back-off from the empty history (KenLM's score with
 * bos = eos = False), summed in fp64 in a fixed order that depends on the row alone and rounded once; w_i is the word of
 * ids[b][i] for i < L and w_L that of the last target, token 0 being </s>, or <s> at position 0.  A token outside [0, V)
 * or a length outside [1, U] makes that row's out NaN; device values are not checked on the host.  The LM must list <s>
 * and </s> ("ngram_score: the LM lists no ..." before any launch otherwise). */
int ccb_ngram_score(const void *lm, int R, int U, const void *ids, long ids_stride, int ids_i64, const void *last,
                    long last_stride, int last_i64, const void *lens, int lens_i64, float *out, void *stream);
/* The rows of a weighted mix of LMs (LODR and the like: DESIGN.md §7 "RNN-T beam search with an LM mix") for
 * ccb_rnnt_beam_step_fused: for every slot q of N*beam, rows[q][k] (V fp32) = sum over the members i, in the given order,
 * of w_i LM_i[q][k], each product and sum rounded in fp64 on its own, the first product starting the sum, rounded to fp32
 * once; -inf if any member's entry is -inf.  The members are n_ngram token n-gram LMs (ccb_ngram_create; ngrams[j],
 * weight ngram_w[j], (N, beam) int32 state arrays state_in[j] and state_out[j]) and n_neural row blocks (neural_rows[j],
 * (N*beam, V) in the CCB_DTYPE_* code neural_dtype[j], weight neural_w[j]); the pointer and weight arrays are host arrays.
 * order[i] (a permutation of 0 .. K-1, K = n_ngram + n_neural) is the i-th member: n-gram order[i] if it is below n_ngram,
 * else neural row block order[i] - n_ngram.  An n-gram member's state and row are those of ccb_ngram_slot_rows with the
 * same parent, token and state arrays (parent null: the start state; token and state_in then unused), and it contributes
 * the fp32 value that entry writes; a neural member's entry is widened exactly.  1 <= K <= 8, weights finite and non-zero,
 * every LM loaded for V labels, and 8 (W + V) bytes at most 200 KiB, W the largest n-gram member's word count. */
int ccb_lm_mix_slot_rows(int n_ngram, const void *const *ngrams, const double *ngram_w, const int *const *state_in,
                         int *const *state_out, int n_neural, const void *const *neural_rows, const int *neural_dtype,
                         const double *neural_w, const int *order, int N, int beam, int V, const int *parent,
                         const int *token, float *rows, void *stream);

/* CTC-T (CTC-Transducer) prefix beam search, one launch per frame, with the arguments and slot arrays of the transducer beam
 * search above; every frame emits one symbol, as in ccb_ctct_forward.  Each live slot holds a prefix with masses b (last
 * emission blank, or none yet) and n (last emission its last token) in the workspace; its score is s = b (+) n.
 *   ccb_ctct_beam_init: the beam [empty prefix, b = -inf, n = 0] and an empty trie.
 *   ccb_ctct_beam_step (frame t; utterances with t >= len_dev[n] keep their beam, each slot its own parent, token -1): rows
 *     and modes as ccb_rnnt_beam_step.  Row r's candidate tokens C_r are the k = min(beam, V - 1) non-blank tokens with the
 *     largest lp_r (ties: lower token).  Extension (r, j), c = C_r[j], adds (c == last_r ? b_r : s_r) + lp_r[c] to
 *     n(prefix_r + c); the stay of r adds s_r + lp_r[blank] to b(prefix_r) and, for a non-empty prefix, n_r + lp_r[last_r]
 *     to n(prefix_r); logaddexp in fp64.  Keys: r (k + 1) + j for an extension, r (k + 1) + k for a stay; a target's key is
 *     its smallest.  The min(beam, #targets with s > -inf) best targets by s desc then key asc form the new beam in that
 *     order: parent slot, token (c for a new extension, -1 for a stay or an extension merged into one), trie node, s.  Dead
 *     slots as in ccb_rnnt_beam_step.  V <= 2^24, blank in [0, V).
 *   ccb_rnnt_beam_finish is the finish for a CTC-T workspace: the beam is already ranked, and the trie comes first in it.
 * workspace: ccb_ctct_beam_ws_bytes(N, Tmax, beam) bytes (0 for beam outside [1, 128]): ccb_rnnt_beam_ws_bytes(N, Tmax,
 * beam) for the tries, then per utterance b and n of every slot and the beam x beam candidate tokens, masses and merges. */
size_t ccb_ctct_beam_ws_bytes(int N, int Tmax, int beam);
int ccb_ctct_beam_init(int N, int Tmax, int beam, void *workspace, int *parent, int *token, int *node, double *score,
                       void *stream);
int ccb_ctct_beam_step(const void *rows, const void *enc, int dtype, int mode, int N, int Tmax, int beam, int V, int t,
                       const int *len_dev, int blank, void *workspace, int *parent, int *token, int *node, double *score,
                       void *stream);

/* number of kernels launched by this library since load (bench.py's gpu_launches) */
long ccb_launch_count(void);

/* Profiling aid: when dev_buffer != NULL the den kernels record, for frames [step0, step0+nsteps) of each pass,
 * per warp chunk 4 x u64 {globaltimer at frame start, clock64 at frame start, clock64 at chunk done, clock64 after
 * the grid barrier} into dev_buffer[(frame-step0) * n_chunks + chunk][4].  Pass NULL to switch it off. */
void ccb_debug_timeline(void *dev_buffer, int step0, int nsteps);

/* ------------------------------------------------------------------------------------------------
 * Section 3 -- host-side den-graph plan (no GPU needed)
 * ---------------------------------------------------------------------------------------------- */
/* Parse + plan without touching CUDA.  n_ctas/n_warps describe the persistent grid the plan is cut for. */
void *ccb_plan_create(const char *fst_name, int n_ctas, int n_warps);
void ccb_plan_destroy(void *plan);
/* info[0..12] = S_file, A_file, S, A_fwd, A_bwd, start, num_labels, n_ctas, n_warps, max_tile_arcs, P (pairs), n_start_arcs,
 *               n_hubs (states whose forward row is split into parts) */
int ccb_plan_info(void *plan, long *info);
/* which: 0 state_label[S] i32, 1 final_lin[S] f32, 2 orig_state[S] i32,
 *        3 fwd_arcs[A_fwd] {u32 peer, f32 w (sign bits = segment events)}, 4 fwd_chunk_state[n_ctas*n_warps+1] i32,
 *        5 fwd_chunk_arc[n_ctas*n_warps+1] i32, 6 bwd_arcs[A_bwd], 7 bwd_chunk_state, 8 bwd_chunk_arc,
 *        9 state_pos[S] i32, 10 fwd_chunk_pair, 11 bwd_chunk_pair, 12 start_arcs[n_start_arcs],
 *        13 fwd_cta_labels[n_ctas*4] i32, 14 bwd_cta_labels, 15 bwd second weights f32[A_bwd], 16 hub_states[n_hubs] i32,
 *        17 / 18 own-row coefficients f32[2S] of the forward / backward pass,
 *        19 in_off[S+1] i32, 20 in_src[A] i32, 21 in_w[A] f32: the in-arc CSR of the split graph the sampler walks (every arc
 *        once, A = in_off[S], linear weights),
 *        22 out_off[S+1] i32, 23 out_dst[A] i32, 24 out_w[A] f32: the same arcs as an out-arc CSR, each state's arcs sorted
 *        by the label of their destination (the beam search's table) */
int ccb_plan_copy(void *plan, int which, void *dst, size_t dst_bytes);
/* The CTC-shape check of ccb_ctc_beam_search(crf=1) on a plan: 0 if it holds, 1 if not (ccb_last_error names the states) */
int ccb_plan_ctc_shape(void *plan);
/* The den kernel launch chosen for one pass (backward 0 / 1) of N utterances at smem_optin bytes of shared memory per block;
 * hooks: bit 0 CCB_ARCS_IN_GLOBAL, 1 CCB_W1_IN_GLOBAL, 2 CCB_NO_TMA, 3 CCB_OWN_IN_L2.  out[0..14] = tier (0 arcs in shared
 * memory, 1 from L2, 2 streamed, 3 small batch), lanes per row, U, batch, w1_smem, Npad, tile_rows, gacc_rows and the
 * shared-memory offsets arcs, ring, bar, w1, abar, aring, total (den_launch.h DenLaunch).  Non-zero: no kernel runs the pass. */
int ccb_plan_launch(void *plan, int N, int backward, int smem_optin, int hooks, long *out);
/* The same launch's own rows: out[0] = 1 if the pass keeps each warp's own rows of the last frame in shared memory (0: it
 * re-reads them from L2), out[1] = their byte offset in dynamic shared memory ([tile_rows][Npad] floats, up to total). */
int ccb_plan_launch_own(void *plan, int N, int backward, int smem_optin, int hooks, long *out);

#ifdef __cplusplus
}
#endif
#endif /* CTC_CRF_B200_H_ */
