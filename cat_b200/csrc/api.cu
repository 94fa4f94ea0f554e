// C ABI of the library (include/ctc_crf_b200.h): den-graph lifetime, workspace carving, launch sequencing.
// Mirrors the roles of the reference's binding.cpp:51-117 + den_calculate.cu:288-481 host code +
// gpu_ctc/ctc_entrypoint.cu:29-109, without torch and without ever calling exit().
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/ctc_crf_b200.h"
#include "common.cuh"
#include "ngram.h"
#include "wfst.h"

using namespace ccb;

int DEN_NUM_ARCS = 0;
int DEN_NUM_STATES = 0;

namespace {

constexpr int kMaxDevices = 64;
thread_local std::string g_err;
std::mutex g_mu;
DenPlan g_plan;                       // host copy (one den graph per process, like den_calculate.cu:263-273)
bool g_plan_valid = false;
DeviceGraph g_dev[kMaxDevices];
int g_refs[kMaxDevices] = {0};        // Init() calls not yet matched by Release(), per device: `ctx = CRFContext(new_graph)` runs the
                                      // old context's __del__ AFTER the new Init -- that Release must not free the new graph
std::atomic<long> g_launches{0};

// scratch owned by the library for the reference-signature entry points (Section 1)
struct LegacyScratch {
    void *aux = nullptr; size_t aux_bytes = 0;
    float *alpha = nullptr; size_t alpha_floats = 0;
    void *ctc = nullptr; size_t ctc_bytes = 0;
    int N = 0, T = 0;
    bool fwd_valid = false;            // compute_alpha ran and compute_beta_and_grad has not consumed it yet
    cudaStream_t stream = nullptr;     // stream the scratch was last allocated / used on (stream-ordered allocation)
    bool used = false;
};
LegacyScratch g_legacy[kMaxDevices];

// profiling aid (ccb_debug_timeline)
unsigned long long *g_timeline = nullptr;
int g_tl_step0 = 0, g_tl_steps = 0;

int Fail(const std::string &m) { g_err = m; return 1; }
int FailCuda(const char *what, cudaError_t e) { g_err = std::string(what) + ": " + cudaGetErrorString(e); return (int)e ? (int)e : 1; }

// the logits dtypes the kernels read (common.cuh load_y); any other code is refused before a kernel sees it
bool KnownDtype(int dtype) { return dtype == CCB_DTYPE_F32 || dtype == CCB_DTYPE_BF16 || dtype == CCB_DTYPE_F16; }
int FailDtype(const char *what, int dtype) {
    return Fail(std::string(what) + ": unsupported logits dtype code " + std::to_string(dtype) +
                " (CCB_DTYPE_F32 0, CCB_DTYPE_BF16 1, CCB_DTYPE_F16 2)");
}

#define CCB_CUDA(call)                                                   \
    do {                                                                 \
        cudaError_t e__ = (call);                                        \
        if (e__ != cudaSuccess) return FailCuda(#call, e__);             \
    } while (0)

template <typename T>
int Upload(T **dst, const std::vector<T> &src) {
    CCB_CUDA(cudaMalloc((void **)dst, std::max<size_t>(src.size(), 1) * sizeof(T)));
    if (!src.empty()) CCB_CUDA(cudaMemcpy(*dst, src.data(), src.size() * sizeof(T), cudaMemcpyHostToDevice));
    return 0;
}

void FreeDevice(DeviceGraph &d) {
    if (!d.loaded) return;
    cudaFree(d.state_label); cudaFree(d.state_pos); cudaFree(d.final_lin); cudaFree(d.start_arcs); cudaFree(d.hub_states);
    for (DevicePass *p : {&d.fwd, &d.bwd}) { cudaFree(p->arcs); cudaFree(p->chunk_state); cudaFree(p->chunk_arc); cudaFree(p->chunk_pair); cudaFree(p->cta_labels); cudaFree(p->w1); cudaFree(p->tq); cudaFree(p->own_c); }
    cudaFree(d.in_off); cudaFree(d.in_src); cudaFree(d.in_w);
    cudaFree(d.out_off); cudaFree(d.out_dst); cudaFree(d.out_w);
    d = DeviceGraph();
}

int UploadPass(const PassPlan &h, DevicePass *d) {
    return Upload(&d->arcs, h.arcs) || Upload(&d->chunk_state, h.chunk_state) || Upload(&d->chunk_arc, h.chunk_arc) ||
           Upload(&d->chunk_pair, h.chunk_pair) || Upload(&d->cta_labels, h.cta_labels) || Upload(&d->w1, h.w1);
}

// The backward pass's quads as the streamed-arc TMA kernel reads them (DevicePass::tq): per quad {row coordinate of slot 0..3}
// {first-weight bits 0..3}{second-weight bits 0..3}; padding slots (both weights zero) name an out-of-bounds row, which the
// TMA unit zero-fills without a fetch.
int UploadTransposedQuads(const PassPlan &h, DevicePass *d) {
    const size_t nq = h.arcs.size() / kQuad;
    std::vector<uint4> tq(nq * 3);
    for (size_t i = 0; i < nq; ++i) {
        uint32_t c[kQuad], w0[kQuad], w1[kQuad];
        for (int j = 0; j < kQuad; ++j) {
            const Arc &a = h.arcs[i * kQuad + j];
            memcpy(&w0[j], &a.w, 4);
            memcpy(&w1[j], &h.w1[i * kQuad + j], 4);
            c[j] = ((w0[j] & 0x7fffffffu) == 0u && w1[j] == 0u) ? kOobRow : (uint32_t)a.peer;
        }
        tq[3 * i] = make_uint4(c[0], c[1], c[2], c[3]);
        tq[3 * i + 1] = make_uint4(w0[0], w0[1], w0[2], w0[3]);
        tq[3 * i + 2] = make_uint4(w1[0], w1[1], w1[2], w1[3]);
    }
    return Upload(&d->tq, tq);
}

int CurrentGraph(DeviceGraph **out) {
    int dev = 0;
    CCB_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= kMaxDevices || !g_dev[dev].loaded)
        return Fail("den graph not loaded on CUDA device " + std::to_string(dev) + " (call Init / CRFContext first)");
    *out = &g_dev[dev];
    return 0;
}

int InitImpl(const char *fst_name, int n_gpus, const int *gpus) {
    std::lock_guard<std::mutex> lk(g_mu);
    if (!fst_name || n_gpus <= 0 || !gpus) return Fail("Init: bad arguments");
    HostFst fst;
    std::string err;
    if (!ReadFstFile(fst_name, &fst, &err)) return Fail(err);
    int prev = 0;
    CCB_CUDA(cudaGetDevice(&prev));
    int count = 0;
    CCB_CUDA(cudaGetDeviceCount(&count));
    for (int i = 0; i < n_gpus; ++i)
        if (gpus[i] < 0 || gpus[i] >= count || gpus[i] >= kMaxDevices) return Fail("Init: invalid GPU id " + std::to_string(gpus[i]));
    cudaDeviceProp prop;
    CCB_CUDA(cudaGetDeviceProperties(&prop, gpus[0]));
    if (!prop.cooperativeLaunch) return Fail("device does not support cooperative launch");
    int n_ctas = prop.multiProcessorCount;
    if (const char *e = getenv("CCB_DEN_CTAS")) {   // test hook: the plan (and grid) of a part with fewer SMs
        char *end = nullptr;
        const long v = strtol(e, &end, 10);
        if (end == e || *end != '\0' || v < 1 || v > prop.multiProcessorCount)
            return Fail(std::string("Init: CCB_DEN_CTAS=") + e + " is not a CTA count in [1, " +
                        std::to_string(prop.multiProcessorCount) + "] (the device's SM count)");
        n_ctas = (int)v;
    }
    if (!BuildDenPlan(fst, n_ctas, kDenThreads / 32, &g_plan, &err)) return Fail(err);
    g_plan_valid = true;
    DEN_NUM_STATES = g_plan.num_states + g_plan.num_pairs;   // rows per alpha frame (what binding.cpp sizes scratch with)
    DEN_NUM_ARCS = (int)g_plan.fwd.arcs.size();
    // the sampler's in-arc CSR and the beam search's out-arc CSR stay on the host until a call needs them on a device
    // (UploadSampleCsr, EnsureBeamGraph)
    auto csr = std::make_shared<DenPlan>();
    csr->in_off = g_plan.in_off; csr->in_src = g_plan.in_src; csr->in_w = g_plan.in_w;
    csr->out_off = g_plan.out_off; csr->out_dst = g_plan.out_dst; csr->out_w = g_plan.out_w;
    csr->num_states = g_plan.num_states; csr->start = g_plan.start;
    csr->state_label = g_plan.state_label; csr->orig_state = g_plan.orig_state;
    int rc = 0;
    for (int i = 0; i < n_gpus && rc == 0; ++i) {
        DeviceGraph &d = g_dev[gpus[i]];
        CCB_CUDA(cudaSetDevice(gpus[i]));
        FreeDevice(d);
        cudaDeviceProp p2;
        CCB_CUDA(cudaGetDeviceProperties(&p2, gpus[i]));
        if (p2.multiProcessorCount != prop.multiProcessorCount) { rc = Fail("Init: heterogeneous GPUs are not supported"); break; }
        d.device = gpus[i];
        d.S = g_plan.num_states; d.P = g_plan.num_pairs; d.start = g_plan.start; d.num_labels = g_plan.num_labels;
        d.scale_exp = g_plan.scale_exp;
        d.n_ctas = g_plan.n_ctas;
        d.max_smem_optin = (int)p2.sharedMemPerBlockOptin;
        rc = Upload(&d.state_label, g_plan.state_label) || Upload(&d.state_pos, g_plan.state_pos) ||
             Upload(&d.final_lin, g_plan.final_lin) || Upload(&d.start_arcs, g_plan.start_arcs) ||
             Upload(&d.hub_states, g_plan.hub_states) ||
             UploadPass(g_plan.fwd, &d.fwd) || UploadPass(g_plan.bwd, &d.bwd) ||
             Upload(&d.fwd.own_c, g_plan.own_fwd) || Upload(&d.bwd.own_c, g_plan.own_bwd);
        d.own_rows = g_plan.own_rows;
        auto on = [](const char *name) { const char *e = getenv(name); return e && e[0] == '1'; };
        d.hooks.arcs_in_global = on("CCB_ARCS_IN_GLOBAL"); d.hooks.w1_in_global = on("CCB_W1_IN_GLOBAL"); d.hooks.no_tma = on("CCB_NO_TMA");
        d.hooks.own_in_l2 = on("CCB_OWN_IN_L2");
        d.shape = ShapeOf(g_plan, d.hooks);
        if (rc == 0 && d.shape.streamed_quads) rc = UploadTransposedQuads(g_plan.bwd, &d.bwd);
        if (d.hooks.arcs_in_global || d.hooks.w1_in_global)
            fprintf(stderr, "ctc_crf_b200: CCB_ARCS_IN_GLOBAL / CCB_W1_IN_GLOBAL set -- den arc tiles forced out of shared memory (test hook, slow)\n");
        d.small_ok = SmallBatchOk(d.shape, d.max_smem_optin, d.hooks);
        d.n_start_arcs = (int)g_plan.start_arcs.size();
        d.start_final = g_plan.final_lin[(size_t)g_plan.start];
        d.host_plan = csr;
        d.loaded = (rc == 0);
        if (rc == 0) ++g_refs[gpus[i]];
    }
    cudaSetDevice(prev);
    return rc;
}

int ReleaseImpl(int n_gpus, const int *gpus) {
    std::lock_guard<std::mutex> lk(g_mu);
    int prev = 0;
    cudaGetDevice(&prev);
    for (int i = 0; i < n_gpus; ++i) {
        if (gpus[i] < 0 || gpus[i] >= kMaxDevices) continue;
        if (g_refs[gpus[i]] > 0 && --g_refs[gpus[i]] > 0) continue;   // a newer Init() still owns this device's graph
        if (cudaSetDevice(gpus[i]) != cudaSuccess) continue;
        cudaDeviceSynchronize();
        FreeDevice(g_dev[gpus[i]]);
        LegacyScratch &ls = g_legacy[gpus[i]];
        cudaFree(ls.aux); cudaFree(ls.alpha); cudaFree(ls.ctc);
        ls = LegacyScratch();
    }
    cudaSetDevice(prev);
    return 0;
}

DenParams BaseParams(const DeviceGraph &g, const void *y, int dtype, long sn, long st, int N, int T, int V,
                     const int *len, float *alpha, void *aux, const DenAuxLayout &L) {
    DenParams p;
    memset(&p, 0, sizeof(p));
    char *a = reinterpret_cast<char *>(aux);
    p.state_label = g.state_label; p.state_pos = g.state_pos; p.final_lin = g.final_lin;
    p.start_arcs = g.start_arcs; p.n_start_arcs = g.n_start_arcs;
    p.hub_states = g.hub_states; p.n_hubs = g.shape.n_hubs;
    p.S = g.S; p.num_pairs = g.P; p.start = g.start; p.n_warps = g.shape.n_warps;
    p.scale_exp = g.scale_exp;
    p.start_final = g.start_final;
    p.y = y; p.y_dtype = dtype; p.sn = sn; p.st = st;
    p.N = N; p.Npad = L.Npad; p.Tmax = T; p.V = V; p.len = len;
    p.alpha = alpha;
    p.a_frames = T + 1 + (g.P > 0 ? 2 : 0);   // full spill (a_base = a_ring = 0: frame t at position t)
    p.t_lo = 0; p.t_hi = T;
    p.bh = reinterpret_cast<float *>(a + L.bh);
    p.colsum_a = reinterpret_cast<float *>(a + L.colsum_a);
    p.colsum_b = reinterpret_cast<float *>(a + L.colsum_b);
    p.absum = reinterpret_cast<float *>(a + L.absum);
    p.zsum = reinterpret_cast<float *>(a + L.zsum);
    p.b0 = reinterpret_cast<float *>(a + L.b0);
    p.fmax = reinterpret_cast<float *>(a + L.fmax);
    p.timeline = g_timeline; p.tl_step0 = g_tl_step0; p.tl_steps = g_tl_steps;
    return p;
}

int CheckDen(const DeviceGraph &g, int dtype, int N, int T, int V) {
    if (N <= 0 || T <= 0 || V <= 0) return Fail("den: empty batch");
    if (!KnownDtype(dtype)) return FailDtype("den", dtype);
    if (V < g.num_labels)
        return Fail("den graph uses label " + std::to_string(g.num_labels - 1) + " but logits have only " + std::to_string(V) + " classes");
    if ((size_t)(2 * (size_t)g.S + g.P) * (size_t)PadLanes(N, g.small_ok) * 4 >= ((size_t)1 << 32)) return Fail("den: states x batch too large for 32-bit row offsets; split the batch");
    if (PadLanes(N, g.small_ok) > g.shape.n_warps * 32) return Fail("den: batch larger than " + std::to_string(g.shape.n_warps * 32) + " utterances per call; split the batch");
    return 0;
}

// Checkpointed alpha (ckpt_k = K > 0): the workspace holds CkptSegFrames positions (the first pass's ring, later one
// segment of frames), then CkptCount checkpoint frames, then the backward pass's carried log-scales (Npad doubles).
void SetCkpt(DenParams &p, const DeviceGraph &g, int T, int K) {
    const size_t frame = (size_t)g.S * p.Npad;
    p.ckpt_k = CkptK(T, K);
    p.ckpt = p.alpha + (size_t)CkptSegFrames(T, K) * frame;
    p.runlog_b = reinterpret_cast<double *>(p.ckpt + (size_t)CkptCount(T, K) * frame);
}

// Forward-only loss: the first checkpointed pass with ckpt_k = T, so frame 0 is the only checkpoint; it sits right behind
// the kAlphaRing + 2 ring positions (ccb_den_fwd_alpha_floats).  No backward pass follows: no carried log-scales.
void SetFwdOnly(DenParams &p, const DeviceGraph &g, int T) {
    p.ckpt_k = T;
    p.ckpt = p.alpha + (size_t)(kAlphaRing + 2) * g.S * p.Npad;
    p.runlog_b = nullptr;
}

// forward part: zero aux, frame max, alpha recursion; logz_a lands in aux
// raw: `y` holds unnormalised logits; the log-normalisers go to aux (lz, lnorm) and logZ comes out normalised
// ckpt_k > 0: alpha on a ring of kAlphaRing frames, checkpoints every ckpt_k frames (see SetCkpt)
// fwd_only: alpha on the ring, logZ only (see SetFwdOnly; ckpt_k is ignored)
int DenForward(const DeviceGraph &g, const void *y, int dtype, long sn, long st, int N, int T, int V, const int *len,
               float *alpha, void *aux, cudaStream_t stream, bool raw = false, int ckpt_k = 0, bool fwd_only = false) {
    const DenAuxLayout L = MakeDenAuxLayout(g.S, N, T, g.small_ok);
    char *a = reinterpret_cast<char *>(aux);
    CCB_CUDA(cudaMemsetAsync(a, 0, L.zero_bytes, stream));
    int rc = raw ? LaunchFrameLse(y, dtype, sn, st, N, T, V, len, reinterpret_cast<float *>(a + L.fmax),
                                  reinterpret_cast<float *>(a + L.lz), reinterpret_cast<double *>(a + L.lnorm), L.Npad, stream)
                 : LaunchFrameMax(y, dtype, sn, st, N, T, V, len, reinterpret_cast<float *>(a + L.fmax), L.Npad, stream);
    if (rc) return FailCuda("frame_max", (cudaError_t)rc);
    DenParams p = BaseParams(g, y, dtype, sn, st, N, T, V, len, alpha, aux, L);
    if (raw) p.lnorm = reinterpret_cast<const double *>(a + L.lnorm);
    p.barrier = reinterpret_cast<unsigned *>(a + L.barrier);
    p.logz = reinterpret_cast<float *>(a + L.logz_a);
    if (ckpt_k > 0 || fwd_only) {
        if (fwd_only) SetFwdOnly(p, g, T);
        else SetCkpt(p, g, T, ckpt_k);
        p.ckpt_mode = 1; p.a_ring = kAlphaRing; p.a_frames = kAlphaRing + 2;
    }
    std::string err;
    rc = LaunchDen(false, g, p, stream, &err);
    if (rc) return Fail(err);
    return 0;
}

// Checkpointed alpha: recompute the frames (lo, hi] of segment j from its checkpoint into the segment positions (frame t at
// position t - lo), as a forward launch that writes neither column sums nor logZ.  Returns lo and hi.
int DenRecompute(const DeviceGraph &g, const void *y, int dtype, long sn, long st, int N, int T, int V, const int *len,
                 float *alpha, void *aux, const DenAuxLayout &L, int ckpt_k, int j, int *lo_out, int *hi_out,
                 cudaStream_t stream) {
    char *a = reinterpret_cast<char *>(aux);
    DenParams f = BaseParams(g, y, dtype, sn, st, N, T, V, len, alpha, aux, L);
    SetCkpt(f, g, T, ckpt_k);
    const int lo = j * f.ckpt_k, hi = std::min(lo + f.ckpt_k, T);
    f.ckpt_mode = 2; f.a_base = lo; f.a_frames = CkptSegFrames(T, ckpt_k);
    f.t_lo = lo; f.t_hi = hi;
    f.barrier = reinterpret_cast<unsigned *>(a + L.barrier);
    CCB_CUDA(cudaMemsetAsync(a + L.barrier, 0, 128, stream));
    std::string err;
    if (LaunchDen(false, g, f, stream, &err)) return Fail(err);
    *lo_out = lo; *hi_out = hi;
    return 0;
}

// backward part (beta recursion, occupancies, logz_b).  ckpt_k > 0: one segment of ckpt_k frames at a time, from the last
// to the first, each first recomputed from its checkpoint into the segment positions by a forward launch.
int DenBackward(const DeviceGraph &g, const void *y, int dtype, long sn, long st, int N, int T, int V, const int *len,
                float *alpha, void *aux, float *grad, long gsn, long gst, float grad_scale, cudaStream_t stream,
                bool raw = false, int ckpt_k = 0) {
    const DenAuxLayout L = MakeDenAuxLayout(g.S, N, T, g.small_ok);
    char *a = reinterpret_cast<char *>(aux);
    DenParams p = BaseParams(g, y, dtype, sn, st, N, T, V, len, alpha, aux, L);
    if (raw) p.lnorm = reinterpret_cast<const double *>(a + L.lnorm);
    p.barrier = reinterpret_cast<unsigned *>(a + L.barrier + 128);
    p.logz = reinterpret_cast<float *>(a + L.logz_b);
    p.grad = grad; p.gsn = gsn; p.gst = gst;
    // the pass accumulates into colsum_b / absum / b0 and counts on its own barrier word: zero them here, so that a second
    // backward pass over the same forward pass (or a reused aux buffer) starts clean instead of relying on DenForward's memset
    CCB_CUDA(cudaMemsetAsync(a + L.colsum_b, 0, L.zsum - L.colsum_b, stream));
    CCB_CUDA(cudaMemsetAsync(a + L.b0, 0, (size_t)L.Npad * 4, stream));
    std::string err;
    int rc = 0;
    if (ckpt_k <= 0) {
        CCB_CUDA(cudaMemsetAsync(a + L.barrier + 128, 0, 128, stream));
        rc = LaunchDen(true, g, p, stream, &err);
        if (rc) return Fail(err);
    } else {
        SetCkpt(p, g, T, ckpt_k);
        for (int j = CkptCount(T, ckpt_k) - 1; j >= 0; --j) {
            int lo = 0, hi = 0;
            if (DenRecompute(g, y, dtype, sn, st, N, T, V, len, alpha, aux, L, ckpt_k, j, &lo, &hi, stream)) return 1;
            p.a_base = lo; p.t_lo = lo; p.t_hi = hi;   // tau = hi .. lo + 1 (tau = 0 epilogue with the first segment)
            CCB_CUDA(cudaMemsetAsync(a + L.barrier + 128, 0, 128, stream));
            rc = LaunchDen(true, g, p, stream, &err);
            if (rc) return Fail(err);
        }
    }
    rc = LaunchDenGradNormalize(grad, gsn, gst, p.absum, len, N, L.Npad, T, V, grad_scale, stream);
    if (rc) return FailCuda("den_grad_normalize", (cudaError_t)rc);
    return 0;
}

// Scratch of the reference-signature route, taken STREAM-ORDERED from the device's default memory pool
// (cudaMallocAsync / cudaFreeAsync on the caller's stream): growing it never synchronises the device.  It is kept
// between calls and returned by Release().  If the caller moves to another stream the old stream is drained first.
int GrowAsync(void **ptr, size_t *have, size_t need, cudaStream_t s) {
    if (*have >= need) return 0;
    if (*ptr) CCB_CUDA(cudaFreeAsync(*ptr, s));
    *ptr = nullptr; *have = 0;
    CCB_CUDA(cudaMallocAsync(ptr, need, s));
    *have = need;
    return 0;
}

int EnsureLegacy(int dev, const DeviceGraph &g, int N, int T, float *caller_alpha, size_t caller_floats, float **alpha_out,
                 cudaStream_t s) {
    LegacyScratch &ls = g_legacy[dev];
    if (ls.used && ls.stream != s) CCB_CUDA(cudaStreamSynchronize(ls.stream));
    ls.stream = s; ls.used = true;
    const DenAuxLayout L = MakeDenAuxLayout(g.S, N, T, g.small_ok);
    if (GrowAsync(&ls.aux, &ls.aux_bytes, L.total, s)) return 1;
    const size_t need = ccb_den_alpha_floats(N, T);
    if (caller_alpha && caller_floats >= need) { *alpha_out = caller_alpha; return 0; }
    size_t have_bytes = ls.alpha_floats * sizeof(float);
    void *ap = ls.alpha;
    if (GrowAsync(&ap, &have_bytes, need * sizeof(float), s)) { ls.alpha = nullptr; ls.alpha_floats = 0; return 1; }
    ls.alpha = reinterpret_cast<float *>(ap); ls.alpha_floats = have_bytes / sizeof(float);
    *alpha_out = ls.alpha;
    return 0;
}

// The RNN-T (CTCT = false) and CTC-T (CTCT = true) entries share their checks and launchers.
template <bool CTCT>
int TransducerForward(const std::string &what, const void *x, int dtype, int from_logits, int compact, int N, long rows, int V,
                      int Tmax, int Umax, const int *labels_dev, long n_labels, const int *lx_dev, const int *ly_dev, int blank,
                      int want_beta, void *workspace, float *costs, float *costs_beta, void *stream) {
    g_err.clear();
    if (N <= 0 || rows < 0 || V <= 0 || n_labels < 0) return Fail(what + ": N and V must be positive, rows and n_labels >= 0");
    if (!KnownDtype(dtype)) return FailDtype(what.c_str(), dtype);
    if (blank < 0 || blank >= V) return Fail(what + ": blank must lie in [0, V)");
    if (!compact && (Tmax < 1 || Umax < 0 || rows != (long)N * Tmax * (Umax + 1) || n_labels != (long)N * Umax))
        return Fail(what + ": the padded layout needs rows = N Tmax (Umax+1) and n_labels = N Umax");
    if (!x || (n_labels && !labels_dev) || !lx_dev || !ly_dev || !workspace || !costs)
        return Fail(what + ": missing buffer");
    const int rc = TransducerLoss<CTCT>::Forward(x, dtype, from_logits, compact, N, rows, V, Tmax, Umax, labels_dev, n_labels,
                                                 lx_dev, ly_dev, blank, want_beta, workspace, costs, costs_beta,
                                                 (cudaStream_t)stream);
    if (rc) return FailCuda(what.c_str(), (cudaError_t)rc);
    return 0;
}

template <bool CTCT>
int TransducerBackward(const std::string &what, const void *x, int dtype, int from_logits, int N, long rows, int V,
                       const int *labels_dev, int blank, void *workspace, const float *w, void *grad, void *stream) {
    g_err.clear();
    if (N <= 0 || rows < 0 || V <= 0) return Fail(what + ": N and V must be positive, rows >= 0");
    if (!KnownDtype(dtype)) return FailDtype(what.c_str(), dtype);
    if (blank < 0 || blank >= V) return Fail(what + ": blank must lie in [0, V)");
    if ((from_logits && !x) || !workspace || !w || !grad) return Fail(what + ": missing buffer");
    const int rc = TransducerLoss<CTCT>::Backward(x, dtype, from_logits, N, rows, V, labels_dev, blank, workspace, w, grad,
                                                  (cudaStream_t)stream);
    if (rc) return FailCuda(what.c_str(), (cudaError_t)rc);
    return 0;
}

template <bool CTCT>
int SimpleForward(const std::string &what, const void *f, const void *g, int dtype, int N, int Tmax, int Umax, int V,
                  const int *labels_dev, const int *lx_dev, const int *ly_dev, int blank, int want_beta, void *workspace,
                  float *costs, void *stream) {
    g_err.clear();
    if (N <= 0 || Tmax <= 0 || Umax < 0 || V <= 0) return Fail(what + ": N, Tmax and V must be positive, Umax >= 0");
    if (N > 65535) return Fail(what + ": at most 65535 utterances per call");
    if (!KnownDtype(dtype)) return FailDtype(what.c_str(), dtype);
    if (blank < 0 || blank >= V) return Fail(what + ": blank must lie in [0, V)");
    if (!f || !g || (Umax && !labels_dev) || !lx_dev || !ly_dev || !workspace || !costs) return Fail(what + ": missing buffer");
    const int rc = TransducerLoss<CTCT>::SimpleForward(f, g, dtype, N, Tmax, Umax, V, labels_dev, lx_dev, ly_dev, blank,
                                                       want_beta, workspace, costs, (cudaStream_t)stream);
    if (rc) return FailCuda(what.c_str(), (cudaError_t)rc);
    return 0;
}

template <bool CTCT>
int SimpleBackward(const std::string &what, const void *f, const void *g, int dtype, int N, int Tmax, int Umax, int V,
                   const int *labels_dev, int blank, void *workspace, const float *w, void *grad_f, void *grad_g, void *stream) {
    g_err.clear();
    if (N <= 0 || Tmax <= 0 || Umax < 0 || V <= 0) return Fail(what + ": N, Tmax and V must be positive, Umax >= 0");
    if (N > 65535) return Fail(what + ": at most 65535 utterances per call");
    if (!KnownDtype(dtype)) return FailDtype(what.c_str(), dtype);
    if (blank < 0 || blank >= V) return Fail(what + ": blank must lie in [0, V)");
    if (!f || !g || (Umax && !labels_dev) || !workspace || !w || !grad_f || !grad_g) return Fail(what + ": missing buffer");
    const int rc = TransducerLoss<CTCT>::SimpleBackward(f, g, dtype, N, Tmax, Umax, V, labels_dev, blank, workspace, w, grad_f,
                                                        grad_g, (cudaStream_t)stream);
    if (rc) return FailCuda(what.c_str(), (cudaError_t)rc);
    return 0;
}

}  // namespace

namespace ccb {
void CountLaunch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
}  // namespace ccb

extern "C" {

const char *ccb_last_error(void) { return g_err.c_str(); }
long ccb_launch_count(void) { return g_launches.load(); }
void ccb_debug_timeline(void *dev_buffer, int step0, int nsteps) {
    g_timeline = reinterpret_cast<unsigned long long *>(dev_buffer); g_tl_step0 = step0; g_tl_steps = nsteps;
}
int ccb_den_info(long *info) {
    if (!g_plan_valid || !info) return 1;
    info[0] = g_plan.file_states; info[1] = g_plan.file_arcs; info[2] = g_plan.num_states; info[3] = g_plan.num_pairs;
    info[4] = (long)g_plan.fwd.arcs.size(); info[5] = (long)g_plan.bwd.arcs.size();
    info[6] = g_plan.fwd.real_arcs; info[7] = g_plan.bwd.real_arcs;
    return 0;
}
int ccb_den_loaded(int device) { return device >= 0 && device < kMaxDevices && g_dev[device].loaded ? 1 : 0; }

void Init(const char *fst_name, int n_gpus, int *gpus) {
    g_err.clear();
    if (InitImpl(fst_name, n_gpus, gpus) != 0) fprintf(stderr, "ctc_crf_b200 Init failed: %s\n", g_err.c_str());
}

void Release(int n_gpus, int *gpus) { ReleaseImpl(n_gpus, gpus); }

// (S, P) of the graph on the CURRENT device when one is loaded there (devices may hold different graphs if Init was
// called per device with different files), else of the last plan built
static void CurrentSizes(int *S, int *P, bool *small_ok) {
    int dev = -1;
    if (cudaGetDevice(&dev) == cudaSuccess && dev >= 0 && dev < kMaxDevices && g_dev[dev].loaded) {
        *S = g_dev[dev].S; *P = g_dev[dev].P; *small_ok = g_dev[dev].small_ok;
        return;
    }
    cudaGetLastError();
    *S = g_plan_valid ? g_plan.num_states : 0; *P = g_plan_valid ? g_plan.num_pairs : 0; *small_ok = false;
}

size_t ccb_den_alpha_floats(int N, int T) {
    int S, P;
    bool small_ok;
    CurrentSizes(&S, &P, &small_ok);
    // T+1 frames of S real rows; the virtual pair-sum rows of a frame are parked two frames ahead (den_kernels.cu), so two
    // more frames at the end when the plan has pairs
    return (size_t)(T + 1 + (P > 0 ? 2 : 0)) * (size_t)S * (size_t)PadLanes(N, small_ok);
}

size_t ccb_den_ckpt_alpha_floats(int N, int T, int K) {
    if (K <= 0 || T <= 0) return ccb_den_alpha_floats(N, T);
    int S, P;
    bool small_ok;
    CurrentSizes(&S, &P, &small_ok);
    // segment / ring positions + checkpoints of S real rows each, then Npad doubles of carried log-scales
    const size_t npad = (size_t)PadLanes(N, small_ok);
    return ((size_t)CkptSegFrames(T, K) + (size_t)CkptCount(T, K)) * (size_t)S * npad + 2 * npad;
}

size_t ccb_den_fwd_alpha_floats(int N) {
    int S, P;
    bool small_ok;
    CurrentSizes(&S, &P, &small_ok);
    // the ring's kAlphaRing + 2 positions, then the one checkpoint (frame 0) of SetFwdOnly, S real rows each; no T in it
    return (size_t)(kAlphaRing + 2 + 1) * (size_t)S * (size_t)PadLanes(N, small_ok);
}

size_t ccb_num_fwd_only_bytes(int N) { return (size_t)(N > 0 ? N : 0) * sizeof(float); }

size_t ccb_den_aux_bytes(int N, int T) {
    int S, P;
    bool small_ok;
    CurrentSizes(&S, &P, &small_ok);
    return S ? MakeDenAuxLayout(S, N, T, small_ok).total : 0;
}

size_t ccb_ctc_workspace_bytes(int N, int T, int max_label_len) {
    // per utterance: alpha and beta cells [T][2L+1] in double + the fp64 log-likelihood (ctc_kernels.cu)
    // ... and, behind them, N floats for the log-likelihoods of the fused loss (LossFwdImpl: `logp`)
    const size_t per_utt = 2 * (size_t)T * (2 * (size_t)max_label_len + 1) + 1;
    return ((size_t)N * per_utt + 32 + ((size_t)N + 1) / 2) * sizeof(double);
}

void compute_alpha(float *alpha, float *logits, const int batch_size, int T, const int alpha_size,
                   int logits_size, int *input_lengths, float *loglikelihood, void *stream) {
    g_err.clear();
    DeviceGraph *g;
    if (CurrentGraph(&g)) return;
    if (CheckDen(*g, CCB_DTYPE_F32, batch_size, T, logits_size)) return;
    float *al = nullptr;
    const size_t caller = (size_t)(T + 1) * (size_t)batch_size * (size_t)(alpha_size > 0 ? alpha_size : 0);
    cudaStream_t s = (cudaStream_t)stream;
    if (EnsureLegacy(g->device, *g, batch_size, T, alpha, caller, &al, s)) return;
    LegacyScratch &ls = g_legacy[g->device];
    ls.N = batch_size; ls.T = T; ls.fwd_valid = false;
    if (DenForward(*g, logits, CCB_DTYPE_F32, (long)T * logits_size, logits_size, batch_size, T, logits_size,
                   input_lengths, al, ls.aux, s)) return;
    ls.fwd_valid = true;
    const DenAuxLayout L = MakeDenAuxLayout(g->S, batch_size, T, g->small_ok);
    cudaError_t e = cudaMemcpyAsync(loglikelihood, (char *)ls.aux + L.logz_a, sizeof(float) * batch_size, cudaMemcpyDeviceToDevice, s);
    if (e != cudaSuccess) FailCuda("copy logZ", e);
}

void compute_beta_and_grad(float *beta, const float *const alpha, const float *const logits,
                           const float *const alpha_lld, float *grad_storage, float *grad_net,
                           const int batch_size, const int T, const int beta_size, const int logits_size,
                           const int *const input_lengths, float *loglikelihood, void *stream) {
    (void)beta; (void)alpha_lld; (void)grad_storage;
    g_err.clear();
    DeviceGraph *g;
    if (CurrentGraph(&g)) return;
    LegacyScratch &ls = g_legacy[g->device];
    // the backward pass continues from the forward pass's column sums / barrier words in the scratch: exactly one
    // compute_beta_and_grad per compute_alpha, same batch
    if (ls.N != batch_size || ls.T != T || !ls.aux || !ls.fwd_valid) { Fail("compute_beta_and_grad: call compute_alpha on the same batch first (once per backward call)"); return; }
    ls.fwd_valid = false;
    float *al = nullptr;
    const size_t caller = (size_t)(T + 1) * (size_t)batch_size * (size_t)(beta_size > 0 ? beta_size : 0);
    cudaStream_t s = (cudaStream_t)stream;
    if (EnsureLegacy(g->device, *g, batch_size, T, const_cast<float *>(alpha), caller, &al, s)) return;
    if (DenBackward(*g, logits, CCB_DTYPE_F32, (long)T * logits_size, logits_size, batch_size, T, logits_size,
                    input_lengths, al, ls.aux, grad_net, (long)T * logits_size, logits_size, 1.f, s)) return;
    if (loglikelihood) {
        const DenAuxLayout L = MakeDenAuxLayout(g->S, batch_size, T, g->small_ok);
        cudaError_t e = cudaMemcpyAsync(loglikelihood, (char *)ls.aux + L.logz_b, sizeof(float) * batch_size, cudaMemcpyDeviceToDevice, s);
        if (e != cudaSuccess) FailCuda("copy logZ(beta)", e);
    }
}

int ccb_den_forward_backward(const void *logits, int dtype, long sn, long st, int N, int T, int V,
                             const int *len_dev, float *alpha_ws, void *aux_ws, float *grad, long gsn, long gst,
                             float grad_scale, float *logz, float *logz_beta, void *stream) {
    g_err.clear();
    DeviceGraph *g;
    if (CurrentGraph(&g)) return 1;
    if (CheckDen(*g, dtype, N, T, V)) return 1;
    if (!alpha_ws || !aux_ws) return Fail("den: workspace missing");
    cudaStream_t s = (cudaStream_t)stream;
    if (DenForward(*g, logits, dtype, sn, st, N, T, V, len_dev, alpha_ws, aux_ws, s)) return 1;
    const DenAuxLayout L = MakeDenAuxLayout(g->S, N, T, g->small_ok);
    if (logz) CCB_CUDA(cudaMemcpyAsync(logz, (char *)aux_ws + L.logz_a, sizeof(float) * N, cudaMemcpyDeviceToDevice, s));
    if (grad) {
        if (DenBackward(*g, logits, dtype, sn, st, N, T, V, len_dev, alpha_ws, aux_ws, grad, gsn, gst, grad_scale, s)) return 1;
        if (logz_beta) CCB_CUDA(cudaMemcpyAsync(logz_beta, (char *)aux_ws + L.logz_b, sizeof(float) * N, cudaMemcpyDeviceToDevice, s));
    }
    return 0;
}

int ccb_ctc_forward_backward(const void *logits, int dtype, long sn, long st, int N, int T, int V,
                             const int *labels_dev, const int *label_off_dev, const int *label_len_dev,
                             const int *len_dev, int max_label_len, int blank, void *workspace,
                             float *grad, long gsn, long gst, float grad_scale, float *logp, void *stream) {
    g_err.clear();
    if (N <= 0 || T <= 0 || V <= 0 || !logits || !workspace || !logp) return Fail("ctc: bad arguments");
    if (!KnownDtype(dtype)) return FailDtype("ctc", dtype);
    if (blank < 0 || blank >= V) return Fail("ctc: blank label out of range");
    std::string err;
    int rc = LaunchCtc(logits, dtype, sn, st, N, T, V, labels_dev, label_off_dev, label_len_dev,
                       len_dev, max_label_len, blank, reinterpret_cast<float *>(workspace), grad, gsn, gst, grad_scale,
                       logp, nullptr, (cudaStream_t)stream, &err);
    if (rc) return Fail(err);
    return 0;
}

/* CTC-only loss (WARP_CTC_LOSS, ctc_crf/__init__.py:25-56) on the (N,T,V) block in place: one numerator pass, the gradient
 * rows all written by the occupancy kernel (no zero fill), the scalar assembled on the device (no host round trip).
 * grad = null: the forward-only loss (one alpha chain per utterance, no cells written, ctc_ws unused). */
static int CtcLossImpl(const char *what, const void *logits, int dtype, int N, int T, int V, int Tmax,
                       const int *labels_dev, const int *label_off_dev, const int *label_len_dev, const int *len_dev,
                       int max_label_len, int blank, float scale, void *ctc_ws, float *grad, float *loss, float *logp,
                       float *costs, int zero_inf, void *stream) {
    g_err.clear();
    if (N <= 0 || T <= 0 || V <= 0 || !logits || (grad && !ctc_ws) || !loss || !logp)
        return Fail(std::string(what) + ": bad arguments");
    if (Tmax <= 0 || Tmax > T) return Fail(std::string(what) + ": Tmax must lie in [1, T]");
    if (!KnownDtype(dtype)) return FailDtype(what, dtype);
    if (blank < 0 || blank >= V) return Fail("ctc: blank label out of range");
    cudaStream_t s = (cudaStream_t)stream;
    const long sn = (long)T * V, st = V;
    std::string err;
    int rc = grad ? LaunchCtc(logits, dtype, sn, st, N, Tmax, V, labels_dev, label_off_dev, label_len_dev, len_dev,
                              max_label_len, blank, reinterpret_cast<float *>(ctc_ws), grad, sn, st, -scale, logp, nullptr, s,
                              &err, /*overwrite=*/1, /*Tfull=*/T, /*logz=*/nullptr, zero_inf)
                  : LaunchCtcLogp(logits, dtype, sn, st, N, Tmax, V, labels_dev, label_off_dev, label_len_dev, len_dev,
                                  max_label_len, blank, logp, nullptr, s, &err);
    if (rc) return Fail(err);
    rc = LaunchSumScale(logp, N, scale, loss, s, costs, zero_inf);
    if (rc) return FailCuda("sum_scale", (cudaError_t)rc);
    return 0;
}

int ccb_ctc_loss_fwd(const void *logits, int dtype, int N, int T, int V, int Tmax,
                     const int *labels_dev, const int *label_off_dev, const int *label_len_dev, const int *len_dev,
                     int max_label_len, int blank, float scale, void *ctc_ws, float *grad, float *loss, float *logp,
                     void *stream) {
    if (!grad) return Fail("ctc_loss_fwd: bad arguments");
    return CtcLossImpl("ctc_loss_fwd", logits, dtype, N, T, V, Tmax, labels_dev, label_off_dev, label_len_dev, len_dev,
                       max_label_len, blank, scale, ctc_ws, grad, loss, logp, nullptr, 0, stream);
}

int ccb_ctc_loss_costs(const void *logits, int dtype, int N, int T, int V, int Tmax,
                       const int *labels_dev, const int *label_off_dev, const int *label_len_dev, const int *len_dev,
                       int max_label_len, int blank, float scale, void *ctc_ws, float *grad, float *loss, float *logp,
                       float *costs, int zero_inf, void *stream) {
    return CtcLossImpl("ctc_loss_costs", logits, dtype, N, T, V, Tmax, labels_dev, label_off_dev, label_len_dev, len_dev,
                       max_label_len, blank, scale, ctc_ws, grad, loss, logp, costs, zero_inf, stream);
}

int ccb_grad_rows_scale(const float *grad, const float *w, const int *len_dev, int N, int T, int V, void *out, int out_dtype,
                        void *stream) {
    g_err.clear();
    if (N <= 0 || T <= 0 || V <= 0 || !grad || !w || !len_dev || !out) return Fail("grad_rows_scale: bad arguments");
    if (!KnownDtype(out_dtype)) return FailDtype("grad_rows_scale", out_dtype);
    int rc = LaunchGradRowsScale(grad, w, len_dev, N, T, V, out, out_dtype, (cudaStream_t)stream);
    if (rc) return FailCuda("grad_rows_scale", (cudaError_t)rc);
    return 0;
}

size_t ccb_ctc_align_workspace_bytes(int N, int T, int max_label_len) {
    return (size_t)N * (size_t)T * (2 * (size_t)max_label_len + 1) + 256;
}

int ccb_ctc_align(const void *logits, int dtype, long sn, long st, int N, int T, int V,
                  const int *labels_dev, const int *label_off_dev, const int *label_len_dev, const int *len_dev,
                  int max_label_len, int blank, void *workspace, int *align, float *score, void *stream) {
    g_err.clear();
    if (N <= 0 || T <= 0 || V <= 0 || !logits || !workspace || !align) return Fail("ctc_align: bad arguments");
    if (!KnownDtype(dtype)) return FailDtype("ctc_align", dtype);
    if (blank < 0 || blank >= V) return Fail("ctc: blank label out of range");
    std::string err;
    int rc = LaunchCtcViterbi(logits, dtype, sn, st, N, T, V, labels_dev, label_off_dev, label_len_dev, len_dev,
                              max_label_len, blank, reinterpret_cast<unsigned char *>(workspace), align, score, (cudaStream_t)stream, &err);
    if (rc) return Fail(err);
    return 0;
}

static int LossFwdImpl(bool raw, const void *logits, int dtype, int N, int T, int V, int Tmax, int ckpt_k,
                       const int *labels_dev, const int *label_off_dev, const int *label_len_dev,
                       const int *len_dev, int max_label_len, float lamb, float scale,
                       float *alpha_ws, void *aux_ws, void *ctc_ws, float *grad, float *loss, float *parts,
                       float *costs, int zero_inf, void *stream) {
    g_err.clear();
    DeviceGraph *g;
    if (CurrentGraph(&g)) return 1;
    if (Tmax <= 0 || Tmax > T) return Fail("ctc_crf_loss_fwd: Tmax must lie in [1, T]");
    if (ckpt_k < 0) return Fail("ctc_crf_loss_fwd: checkpoint interval must be >= 0");
    if (CheckDen(*g, dtype, N, Tmax, V)) return 1;
    if (!alpha_ws || !aux_ws || !ctc_ws || !grad || !loss) return Fail("ctc_crf_loss_fwd: missing buffer");
    cudaStream_t s = (cudaStream_t)stream;
    const long sn = (long)T * V, st = V;     // the (N,T,V) block is addressed in place; only Tmax frames are walked
    const DenAuxLayout L = MakeDenAuxLayout(g->S, N, Tmax, g->small_ok);
    float *logz = reinterpret_cast<float *>((char *)aux_ws + L.logz_a);
    // log p(l|x) per utterance: the numerator's output, kept behind its cells in ITS workspace (ccb_ctc_workspace_bytes
    // counts it)
    float *logp = reinterpret_cast<float *>(reinterpret_cast<double *>(ctc_ws) +
                                            (size_t)N * (2 * (size_t)Tmax * (2 * (size_t)max_label_len + 1) + 1) + 32);
    const double *lnorm = raw ? reinterpret_cast<const double *>((char *)aux_ws + L.lnorm) : nullptr;
    CCB_CUDA(cudaMemsetAsync(grad, 0, sizeof(float) * (size_t)N * T * V, s));
    if (DenForward(*g, logits, dtype, sn, st, N, Tmax, V, len_dev, alpha_ws, aux_ws, s, raw, ckpt_k)) return 1;
    if (DenBackward(*g, logits, dtype, sn, st, N, Tmax, V, len_dev, alpha_ws, aux_ws, grad, sn, st, scale, s, raw, ckpt_k)) return 1;
    // the numerator accumulates into the gradient after the den passes have normalised their part of it (with zero_inf it
    // overwrites the rows of an utterance whose logZ or log p is not finite with zeros instead)
    std::string err;
    int rc = LaunchCtc(logits, dtype, sn, st, N, Tmax, V, labels_dev, label_off_dev, label_len_dev, len_dev,
                       max_label_len, 0, reinterpret_cast<float *>(ctc_ws), grad, sn, st, -(1.f + lamb) * scale, logp, lnorm, s, &err,
                       /*overwrite=*/0, /*Tfull=*/0, logz, zero_inf);
    if (rc) return Fail(err);
    if (raw) {   // chain through log_softmax: dL/dz = g - softmax(z) * sum_k g_k (a zero row stays zero)
        rc = LaunchLogitGrad(logits, dtype, sn, st, N, Tmax, V, len_dev,
                             reinterpret_cast<const float *>((char *)aux_ws + L.lz), L.Npad, grad, sn, st, s);
        if (rc) return FailCuda("logit_grad", (cudaError_t)rc);
    }
    rc = LaunchAssembleLoss(logz, logp, N, lamb, scale, loss, s, costs, zero_inf);
    if (rc) return FailCuda("assemble_loss", (cudaError_t)rc);
    if (parts) {
        CCB_CUDA(cudaMemcpyAsync(parts, logz, sizeof(float) * N, cudaMemcpyDeviceToDevice, s));
        CCB_CUDA(cudaMemcpyAsync(parts + N, logp, sizeof(float) * N, cudaMemcpyDeviceToDevice, s));
    }
    return 0;
}

int ccb_ctc_crf_loss_fwd(const void *logits, int dtype, int N, int T, int V, int Tmax,
                         const int *labels_dev, const int *label_off_dev, const int *label_len_dev,
                         const int *len_dev, int max_label_len, float lamb, float scale,
                         float *alpha_ws, void *aux_ws, void *ctc_ws, float *grad, float *loss, float *parts,
                         void *stream) {
    return LossFwdImpl(false, logits, dtype, N, T, V, Tmax, 0, labels_dev, label_off_dev, label_len_dev, len_dev, max_label_len,
                       lamb, scale, alpha_ws, aux_ws, ctc_ws, grad, loss, parts, nullptr, 0, stream);
}

int ccb_ctc_crf_loss_logits_fwd(const void *logits, int dtype, int N, int T, int V, int Tmax,
                                const int *labels_dev, const int *label_off_dev, const int *label_len_dev,
                                const int *len_dev, int max_label_len, float lamb, float scale,
                                float *alpha_ws, void *aux_ws, void *ctc_ws, float *grad, float *loss, float *parts,
                                void *stream) {
    return LossFwdImpl(true, logits, dtype, N, T, V, Tmax, 0, labels_dev, label_off_dev, label_len_dev, len_dev, max_label_len,
                       lamb, scale, alpha_ws, aux_ws, ctc_ws, grad, loss, parts, nullptr, 0, stream);
}

int ccb_ctc_crf_loss_ckpt_fwd(const void *logits, int dtype, int N, int T, int V, int Tmax, int ckpt_k,
                              const int *labels_dev, const int *label_off_dev, const int *label_len_dev,
                              const int *len_dev, int max_label_len, float lamb, float scale,
                              float *alpha_ws, void *aux_ws, void *ctc_ws, float *grad, float *loss, float *parts,
                              void *stream) {
    return LossFwdImpl(false, logits, dtype, N, T, V, Tmax, ckpt_k, labels_dev, label_off_dev, label_len_dev, len_dev,
                       max_label_len, lamb, scale, alpha_ws, aux_ws, ctc_ws, grad, loss, parts, nullptr, 0, stream);
}

int ccb_ctc_crf_loss_logits_ckpt_fwd(const void *logits, int dtype, int N, int T, int V, int Tmax, int ckpt_k,
                                     const int *labels_dev, const int *label_off_dev, const int *label_len_dev,
                                     const int *len_dev, int max_label_len, float lamb, float scale,
                                     float *alpha_ws, void *aux_ws, void *ctc_ws, float *grad, float *loss, float *parts,
                                     void *stream) {
    return LossFwdImpl(true, logits, dtype, N, T, V, Tmax, ckpt_k, labels_dev, label_off_dev, label_len_dev, len_dev,
                       max_label_len, lamb, scale, alpha_ws, aux_ws, ctc_ws, grad, loss, parts, nullptr, 0, stream);
}

/* Forward-only CTC-CRF loss: the same loss (and parts) as LossFwdImpl without the gradient.  The den forward pass keeps
 * alpha on the ring (SetFwdOnly), the numerator walks its alpha chains without writing cells, and nothing touches an (N,T,V)
 * buffer but the logits.  Launches: frame max (raw: frame log-sum-exp + normalisers), den forward, numerator, loss. */
static int LossFwdOnlyImpl(bool raw, const void *logits, int dtype, int N, int T, int V, int Tmax,
                           const int *labels_dev, const int *label_off_dev, const int *label_len_dev,
                           const int *len_dev, int max_label_len, float lamb, float scale,
                           float *alpha_ws, void *aux_ws, void *num_ws, float *loss, float *parts, float *costs,
                           int zero_inf, void *stream) {
    g_err.clear();
    DeviceGraph *g;
    if (CurrentGraph(&g)) return 1;
    if (Tmax <= 0 || Tmax > T) return Fail("ctc_crf_loss_fwd_only: Tmax must lie in [1, T]");
    if (CheckDen(*g, dtype, N, Tmax, V)) return 1;
    if (!alpha_ws || !aux_ws || !num_ws || !loss) return Fail("ctc_crf_loss_fwd_only: missing buffer");
    cudaStream_t s = (cudaStream_t)stream;
    const long sn = (long)T * V, st = V;
    const DenAuxLayout L = MakeDenAuxLayout(g->S, N, Tmax, g->small_ok);
    float *logz = reinterpret_cast<float *>((char *)aux_ws + L.logz_a);
    float *logp = reinterpret_cast<float *>(num_ws);
    const double *lnorm = raw ? reinterpret_cast<const double *>((char *)aux_ws + L.lnorm) : nullptr;
    if (DenForward(*g, logits, dtype, sn, st, N, Tmax, V, len_dev, alpha_ws, aux_ws, s, raw, 0, /*fwd_only=*/true)) return 1;
    std::string err;
    int rc = LaunchCtcLogp(logits, dtype, sn, st, N, Tmax, V, labels_dev, label_off_dev, label_len_dev,
                           len_dev, max_label_len, 0, logp, lnorm, s, &err);
    if (rc) return Fail(err);
    rc = LaunchAssembleLoss(logz, logp, N, lamb, scale, loss, s, costs, zero_inf);
    if (rc) return FailCuda("assemble_loss", (cudaError_t)rc);
    if (parts) {
        CCB_CUDA(cudaMemcpyAsync(parts, logz, sizeof(float) * N, cudaMemcpyDeviceToDevice, s));
        CCB_CUDA(cudaMemcpyAsync(parts + N, logp, sizeof(float) * N, cudaMemcpyDeviceToDevice, s));
    }
    return 0;
}

int ccb_ctc_crf_loss_fwd_only(const void *logits, int dtype, int from_logits, int N, int T, int V, int Tmax,
                              const int *labels_dev, const int *label_off_dev, const int *label_len_dev,
                              const int *len_dev, int max_label_len, float lamb, float scale,
                              float *alpha_ws, void *aux_ws, void *num_ws, float *loss, float *parts, void *stream) {
    return LossFwdOnlyImpl(from_logits != 0, logits, dtype, N, T, V, Tmax, labels_dev, label_off_dev, label_len_dev, len_dev,
                           max_label_len, lamb, scale, alpha_ws, aux_ws, num_ws, loss, parts, nullptr, 0, stream);
}

int ccb_ctc_crf_loss_costs(const void *logits, int dtype, int from_logits, int N, int T, int V, int Tmax, int ckpt_k,
                           const int *labels_dev, const int *label_off_dev, const int *label_len_dev,
                           const int *len_dev, int max_label_len, float lamb, float scale,
                           float *alpha_ws, void *aux_ws, void *ctc_ws, float *grad, float *loss, float *parts,
                           float *costs, int zero_inf, void *stream) {
    return LossFwdImpl(from_logits != 0, logits, dtype, N, T, V, Tmax, ckpt_k, labels_dev, label_off_dev, label_len_dev, len_dev,
                       max_label_len, lamb, scale, alpha_ws, aux_ws, ctc_ws, grad, loss, parts, costs, zero_inf, stream);
}

int ccb_ctc_crf_loss_costs_fwd_only(const void *logits, int dtype, int from_logits, int N, int T, int V, int Tmax,
                                    const int *labels_dev, const int *label_off_dev, const int *label_len_dev,
                                    const int *len_dev, int max_label_len, float lamb, float scale,
                                    float *alpha_ws, void *aux_ws, void *num_ws, float *loss, float *parts,
                                    float *costs, int zero_inf, void *stream) {
    return LossFwdOnlyImpl(from_logits != 0, logits, dtype, N, T, V, Tmax, labels_dev, label_off_dev, label_len_dev, len_dev,
                           max_label_len, lamb, scale, alpha_ws, aux_ws, num_ws, loss, parts, costs, zero_inf, stream);
}

int ccb_ctc_loss_fwd_only(const void *logits, int dtype, int N, int T, int V, int Tmax,
                          const int *labels_dev, const int *label_off_dev, const int *label_len_dev, const int *len_dev,
                          int max_label_len, int blank, float scale, float *loss, float *logp, void *stream) {
    return CtcLossImpl("ctc_loss_fwd_only", logits, dtype, N, T, V, Tmax, labels_dev, label_off_dev, label_len_dev, len_dev,
                       max_label_len, blank, scale, nullptr, nullptr, loss, logp, nullptr, 0, stream);
}

/* ---- several label sequences per utterance ------------------------------------------------------ */
static int CheckSeqMap(const char *what, int M, const int *seq_row, const int *seq_pos) {
    // M = 0 is a slice of utterances without sequences: their gradient rows are zeros, their share of the loss 0
    if (M < 0 || (M > 0 && (!seq_row || !seq_pos))) return Fail(std::string(what) + ": bad sequence map");
    return 0;
}

// the numerator's log-likelihoods of M sequences, behind their cells in the numerator workspace (as in LossFwdImpl)
static float *SeqLogp(void *ctc_ws, int M, int Tmax, int max_label_len) {
    return reinterpret_cast<float *>(reinterpret_cast<double *>(ctc_ws) +
                                     (size_t)M * (2 * (size_t)Tmax * (2 * (size_t)max_label_len + 1) + 1) + 32);
}

int ccb_ctc_crf_loss_seqs(const void *logits, int dtype, int from_logits, int N, int T, int V, int Tmax, int ckpt_k,
                          const int *labels_dev, const int *label_off_dev, const int *label_len_dev, const int *len_dev,
                          int M, const int *seq_row_dev, const int *seq_pos_dev, const int *seq_off_dev, int max_label_len,
                          float lamb, float scale, float *alpha_ws, void *aux_ws, void *ctc_ws, float *grad, float *loss,
                          float *costs, int zero_inf, int defer_num, void *stream) {
    g_err.clear();
    const bool raw = from_logits != 0;
    DeviceGraph *g;
    if (CurrentGraph(&g)) return 1;
    if (Tmax <= 0 || Tmax > T) return Fail("ctc_crf_loss_seqs: Tmax must lie in [1, T]");
    if (ckpt_k < 0) return Fail("ctc_crf_loss_seqs: checkpoint interval must be >= 0");
    if (CheckSeqMap("ctc_crf_loss_seqs", M, seq_row_dev, seq_pos_dev) || CheckDen(*g, dtype, N, Tmax, V)) return 1;
    if (!alpha_ws || !aux_ws || !ctc_ws || !grad || !loss || !seq_off_dev) return Fail("ctc_crf_loss_seqs: missing buffer");
    cudaStream_t s = (cudaStream_t)stream;
    const long sn = (long)T * V, st = V;
    const DenAuxLayout L = MakeDenAuxLayout(g->S, N, Tmax, g->small_ok);
    float *logz = reinterpret_cast<float *>((char *)aux_ws + L.logz_a);
    float *logp = SeqLogp(ctc_ws, M, Tmax, max_label_len);
    const double *lnorm = raw ? reinterpret_cast<const double *>((char *)aux_ws + L.lnorm) : nullptr;
    // the den passes run once per utterance and leave its occupancies UNSCALED in grad; the gamma pass scales them by the
    // weight of the utterance's sequences
    CCB_CUDA(cudaMemsetAsync(grad, 0, sizeof(float) * (size_t)N * T * V, s));
    if (DenForward(*g, logits, dtype, sn, st, N, Tmax, V, len_dev, alpha_ws, aux_ws, s, raw, ckpt_k)) return 1;
    if (DenBackward(*g, logits, dtype, sn, st, N, Tmax, V, len_dev, alpha_ws, aux_ws, grad, sn, st, 1.f, s, raw, ckpt_k)) return 1;
    std::string err;
    int rc = LaunchCtcSeqs(logits, dtype, sn, st, M, Tmax, V, labels_dev, label_off_dev, label_len_dev, len_dev, seq_row_dev,
                           max_label_len, 0, reinterpret_cast<float *>(ctc_ws), true, logp, lnorm, s, &err);
    if (rc) return Fail(err);
    if (!defer_num) {
        rc = LaunchCtcGammaSeqs(logits, dtype, sn, st, N, Tmax, T, V, labels_dev, label_off_dev, label_len_dev, len_dev,
                                seq_off_dev, seq_pos_dev, max_label_len, 0, reinterpret_cast<float *>(ctc_ws), nullptr, scale,
                                -(1.f + lamb), grad, logz, zero_inf, grad, sn, st, s, &err);
        if (rc) return Fail(err);
        if (raw) {
            rc = LaunchLogitGrad(logits, dtype, sn, st, N, Tmax, V, len_dev,
                                 reinterpret_cast<const float *>((char *)aux_ws + L.lz), L.Npad, grad, sn, st, s);
            if (rc) return FailCuda("logit_grad", (cudaError_t)rc);
        }
    }
    rc = LaunchSeqCosts(logz, logp, seq_row_dev, seq_pos_dev, M, lamb, scale, loss, costs, zero_inf, s);
    if (rc) return FailCuda("seq_costs", (cudaError_t)rc);
    return 0;
}

int ccb_ctc_crf_loss_seqs_fwd_only(const void *logits, int dtype, int from_logits, int N, int T, int V, int Tmax,
                                   const int *labels_dev, const int *label_off_dev, const int *label_len_dev,
                                   const int *len_dev, int M, const int *seq_row_dev, const int *seq_pos_dev,
                                   int max_label_len, float lamb, float scale, float *alpha_ws, void *aux_ws, void *num_ws,
                                   float *loss, float *costs, int zero_inf, void *stream) {
    g_err.clear();
    const bool raw = from_logits != 0;
    DeviceGraph *g;
    if (CurrentGraph(&g)) return 1;
    if (Tmax <= 0 || Tmax > T) return Fail("ctc_crf_loss_seqs_fwd_only: Tmax must lie in [1, T]");
    if (CheckSeqMap("ctc_crf_loss_seqs_fwd_only", M, seq_row_dev, seq_pos_dev) || CheckDen(*g, dtype, N, Tmax, V)) return 1;
    if (!alpha_ws || !aux_ws || !num_ws || !loss) return Fail("ctc_crf_loss_seqs_fwd_only: missing buffer");
    cudaStream_t s = (cudaStream_t)stream;
    const long sn = (long)T * V, st = V;
    const DenAuxLayout L = MakeDenAuxLayout(g->S, N, Tmax, g->small_ok);
    float *logz = reinterpret_cast<float *>((char *)aux_ws + L.logz_a);
    float *logp = reinterpret_cast<float *>(num_ws);
    const double *lnorm = raw ? reinterpret_cast<const double *>((char *)aux_ws + L.lnorm) : nullptr;
    if (DenForward(*g, logits, dtype, sn, st, N, Tmax, V, len_dev, alpha_ws, aux_ws, s, raw, 0, /*fwd_only=*/true)) return 1;
    std::string err;
    int rc = LaunchCtcSeqs(logits, dtype, sn, st, M, Tmax, V, labels_dev, label_off_dev, label_len_dev, len_dev, seq_row_dev,
                           max_label_len, 0, nullptr, false, logp, lnorm, s, &err);
    if (rc) return Fail(err);
    rc = LaunchSeqCosts(logz, logp, seq_row_dev, seq_pos_dev, M, lamb, scale, loss, costs, zero_inf, s);
    if (rc) return FailCuda("seq_costs", (cudaError_t)rc);
    return 0;
}

int ccb_ctc_loss_seqs(const void *logits, int dtype, int N, int T, int V, int Tmax,
                      const int *labels_dev, const int *label_off_dev, const int *label_len_dev, const int *len_dev,
                      int M, const int *seq_row_dev, const int *seq_pos_dev, const int *seq_off_dev, int max_label_len,
                      int blank, float scale, void *ctc_ws, float *grad, float *loss, float *logp, float *costs,
                      int zero_inf, int defer_num, void *stream) {
    g_err.clear();
    if (N <= 0 || T <= 0 || V <= 0 || !logits || !loss || !logp || (ctc_ws && !defer_num && !grad))
        return Fail("ctc_loss_seqs: bad arguments");
    if (Tmax <= 0 || Tmax > T) return Fail("ctc_loss_seqs: Tmax must lie in [1, T]");
    if (!KnownDtype(dtype)) return FailDtype("ctc_loss_seqs", dtype);
    if (blank < 0 || blank >= V) return Fail("ctc: blank label out of range");
    if (CheckSeqMap("ctc_loss_seqs", M, seq_row_dev, seq_pos_dev)) return 1;
    if (ctc_ws && !defer_num && !seq_off_dev) return Fail("ctc_loss_seqs: missing sequence offsets");
    cudaStream_t s = (cudaStream_t)stream;
    const long sn = (long)T * V, st = V;
    std::string err;
    int rc = LaunchCtcSeqs(logits, dtype, sn, st, M, Tmax, V, labels_dev, label_off_dev, label_len_dev, len_dev, seq_row_dev,
                           max_label_len, blank, reinterpret_cast<float *>(ctc_ws), ctc_ws != nullptr, logp, nullptr, s, &err);
    if (rc) return Fail(err);
    if (ctc_ws && !defer_num) {   // every row of the (N,T,V) gradient is written
        rc = LaunchCtcGammaSeqs(logits, dtype, sn, st, N, Tmax, T, V, labels_dev, label_off_dev, label_len_dev, len_dev,
                                seq_off_dev, seq_pos_dev, max_label_len, blank, reinterpret_cast<float *>(ctc_ws), nullptr,
                                scale, -1.f, nullptr, nullptr, zero_inf, grad, sn, st, s, &err);
        if (rc) return Fail(err);
    }
    rc = LaunchSeqCosts(nullptr, logp, seq_row_dev, seq_pos_dev, M, 0.f, scale, loss, costs, zero_inf, s);
    if (rc) return FailCuda("seq_costs", (cudaError_t)rc);
    return 0;
}

int ccb_seqs_grad(const void *logits, int dtype, int from_logits, int N, int T, int V, int Tmax,
                  const int *labels_dev, const int *label_off_dev, const int *label_len_dev, const int *len_dev,
                  int M, const int *seq_pos_dev, const int *seq_off_dev, int max_label_len, int blank, float num_coef,
                  const float *w, const float *den, void *aux_ws, void *ctc_ws, int zero_inf, float *out, void *stream) {
    g_err.clear();
    const bool raw = from_logits != 0;
    if (N <= 0 || T <= 0 || V <= 0 || M < 0 || !logits || !w || !ctc_ws || !out || !seq_off_dev || (M > 0 && !seq_pos_dev))
        return Fail("seqs_grad: bad arguments");
    if (Tmax <= 0 || Tmax > T) return Fail("seqs_grad: Tmax must lie in [1, T]");
    if (!KnownDtype(dtype)) return FailDtype("seqs_grad", dtype);
    if ((den || raw) && !aux_ws) return Fail("seqs_grad: the den part needs the forward call's aux workspace");
    if (raw && !den) return Fail("seqs_grad: from_logits needs the den part");
    cudaStream_t s = (cudaStream_t)stream;
    const long sn = (long)T * V, st = V;
    const float *logz = nullptr;
    DenAuxLayout L;
    if (den) {
        DeviceGraph *g;
        if (CurrentGraph(&g)) return 1;
        L = MakeDenAuxLayout(g->S, N, Tmax, g->small_ok);
        logz = reinterpret_cast<const float *>((char *)aux_ws + L.logz_a);
    }
    std::string err;
    int rc = LaunchCtcGammaSeqs(logits, dtype, sn, st, N, Tmax, T, V, labels_dev, label_off_dev, label_len_dev, len_dev,
                                seq_off_dev, seq_pos_dev, max_label_len, blank, reinterpret_cast<float *>(ctc_ws), w, 1.f,
                                num_coef, den, logz, zero_inf, out, sn, st, s, &err);
    if (rc) return Fail(err);
    if (raw) {
        rc = LaunchLogitGrad(logits, dtype, sn, st, N, Tmax, V, len_dev,
                             reinterpret_cast<const float *>((char *)aux_ws + L.lz), L.Npad, out, sn, st, s);
        if (rc) return FailCuda("logit_grad", (cudaError_t)rc);
    }
    return 0;
}

int ccb_ctc_align_seqs(const void *logits, int dtype, long sn, long st, int N, int T, int V,
                       const int *labels_dev, const int *label_off_dev, const int *label_len_dev, const int *len_dev,
                       int M, const int *seq_row_dev, const int *seq_pos_dev, int max_label_len, int blank, void *workspace,
                       int *align, float *score, void *stream) {
    g_err.clear();
    if (N <= 0 || T <= 0 || V <= 0 || !logits || !workspace || !align) return Fail("ctc_align_seqs: bad arguments");
    if (!KnownDtype(dtype)) return FailDtype("ctc_align_seqs", dtype);
    if (blank < 0 || blank >= V) return Fail("ctc: blank label out of range");
    if (CheckSeqMap("ctc_align_seqs", M, seq_row_dev, seq_pos_dev)) return 1;
    std::string err;
    int rc = LaunchCtcViterbiSeqs(logits, dtype, sn, st, M, T, V, labels_dev, label_off_dev, label_len_dev, len_dev, seq_row_dev,
                                  seq_pos_dev, max_label_len, blank, reinterpret_cast<unsigned char *>(workspace), align, score,
                                  (cudaStream_t)stream, &err);
    if (rc) return Fail(err);
    return 0;
}

/* ---- samples from the CTC-CRF posterior ------------------------------------------------------ */
// The in-arc CSR of the device's graph, uploaded by the first sampling call on the device (Release frees it with the graph)
static int UploadSampleCsr(DeviceGraph *g) {
    std::lock_guard<std::mutex> lk(g_mu);
    if (g->in_off) return 0;
    if (!g->host_plan) return Fail("crf_sample: the den graph's in-arc table is missing");
    const DenPlan &h = *g->host_plan;
    int *off = nullptr, *src = nullptr;
    float *w = nullptr;
    if (Upload(&off, h.in_off) || Upload(&src, h.in_src) || Upload(&w, h.in_w)) {
        cudaFree(off); cudaFree(src); cudaFree(w);
        return 1;
    }
    g->in_src = src; g->in_w = w; g->in_off = off;
    return 0;
}

size_t ccb_crf_sample_ws_bytes(int N, int K, int T) {
    (void)T;   // the records carry the walk across segments; nothing in the workspace grows with the frames
    int S, P;
    bool small_ok;
    CurrentSizes(&S, &P, &small_ok);
    return N > 0 && K > 0 ? SampleWsBytes(N, K, S) : 0;
}

int ccb_crf_sample(const void *logits, int dtype, int N, int T, int V, int Tmax, int ckpt_k, const int *len_dev, int K,
                   unsigned long long seed, int n_base, float *alpha_ws, void *aux_ws, void *sample_ws, int *tokens,
                   int *lengths, int *align, float *path_logp, void *stream) {
    g_err.clear();
    DeviceGraph *g;
    if (CurrentGraph(&g)) return 1;
    if (Tmax <= 0 || Tmax > T) return Fail("crf_sample: Tmax must lie in [1, T]");
    if (ckpt_k < 0) return Fail("crf_sample: checkpoint interval must be >= 0");
    if (K <= 0 || n_base < 0) return Fail("crf_sample: bad sample count or utterance offset");
    if (CheckDen(*g, dtype, N, Tmax, V)) return 1;
    if (!logits || !len_dev || !alpha_ws || !aux_ws || !sample_ws || !tokens || !lengths || !align || !path_logp)
        return Fail("crf_sample: missing buffer");
    if (UploadSampleCsr(g)) return 1;
    cudaStream_t s = (cudaStream_t)stream;
    const long sn = (long)T * V, st = V;
    const DenAuxLayout L = MakeDenAuxLayout(g->S, N, Tmax, g->small_ok);
    const float *logz = reinterpret_cast<const float *>((char *)aux_ws + L.logz_a);
    // log-probs or raw logits alike: every path emits one label per frame, so a per-frame shift cancels in p(path | x)
    if (DenForward(*g, logits, dtype, sn, st, N, Tmax, V, len_dev, alpha_ws, aux_ws, s, false, ckpt_k)) return 1;
    // frames (lo, hi] of alpha at positions t - lo: the full spill is the one segment (0, Tmax]
    auto walk = [&](int lo, int hi, bool first) -> int {
        int rc = LaunchSampleFinalPrefix(alpha_ws, lo, g->S, L.Npad, g->final_lin, len_dev, N, lo, hi, sample_ws,
                                         K, s);
        if (rc) return FailCuda("sample_final_prefix", (cudaError_t)rc);
        rc = LaunchSampleWalk(*g, logits, dtype, sn, st, N, T, Tmax, L.Npad, len_dev, alpha_ws, lo, lo, hi, first,
                              K, seed, n_base, logz, sample_ws, tokens, lengths, align, path_logp, s);
        if (rc) return FailCuda("sample_walk", (cudaError_t)rc);
        return 0;
    };
    if (ckpt_k <= 0) return walk(0, Tmax, true);
    // checkpointed: each segment is recomputed from its checkpoint and walked, the last one first
    for (int j = CkptCount(Tmax, ckpt_k) - 1; j >= 0; --j) {
        int lo = 0, hi = 0;
        if (DenRecompute(*g, logits, dtype, sn, st, N, Tmax, V, len_dev, alpha_ws, aux_ws, L, ckpt_k, j, &lo, &hi, s)) return 1;
        if (walk(lo, hi, j == CkptCount(Tmax, ckpt_k) - 1)) return 1;
    }
    return 0;
}

/* ---- CTC prefix beam search ------------------------------------------------------------------ */
// A token n-gram LM handle (ccb_ngram_create): the host tables, and their device copies, uploaded by the first search that
// uses the LM on a device and freed by ccb_ngram_destroy
struct NGram {
    NGramHost host;
    bool uploaded[kMaxDevices] = {};
    NGramDev dev[kMaxDevices];
    std::vector<void *> blocks[kMaxDevices];
};

static int EnsureNGram(NGram *m, const NGramDev **out) {
    std::lock_guard<std::mutex> lk(g_mu);
    int d = 0;
    CCB_CUDA(cudaGetDevice(&d));
    if (d < 0 || d >= kMaxDevices) return Fail("ctc_beam_search: CUDA device " + std::to_string(d) + " is out of range");
    if (!m->uploaded[d]) {
        const NGramHost &h = m->host;
        NGramDev t;
        int *tok2word = nullptr, *root_dst = nullptr, *arc_off = nullptr, *arc_word = nullptr, *arc_dst = nullptr, *back = nullptr;
        float *root_p = nullptr, *arc_p = nullptr, *bow = nullptr;
        const int rc = Upload(&tok2word, h.tok2word) || Upload(&root_dst, h.root_dst) || Upload(&arc_off, h.arc_off) ||
                       Upload(&arc_word, h.arc_word) || Upload(&arc_dst, h.arc_dst) || Upload(&back, h.back) ||
                       Upload(&root_p, h.root_p) || Upload(&arc_p, h.arc_p) || Upload(&bow, h.bow);
        m->blocks[d] = {tok2word, root_dst, arc_off, arc_word, arc_dst, back, root_p, arc_p, bow};
        if (rc) {
            for (void *p : m->blocks[d]) cudaFree(p);
            m->blocks[d].clear();
            return 1;
        }
        t.tok2word = tok2word; t.root_dst = root_dst; t.arc_off = arc_off; t.arc_word = arc_word; t.arc_dst = arc_dst;
        t.back = back; t.root_p = root_p; t.arc_p = arc_p; t.bow = bow; t.bos = h.bos; t.eos = h.eos;
        m->dev[d] = t;
        m->uploaded[d] = true;
    }
    *out = &m->dev[d];
    return 0;
}


// crf mode: the CTC-shape check of the device's graph (once; the result is kept) and its out-arc CSR on the device
static int EnsureBeamGraph(DeviceGraph *g) {
    std::lock_guard<std::mutex> lk(g_mu);
    if (g->ctc_shape < 0) {
        if (!g->host_plan) return Fail("ctc_beam_search: the den graph's out-arc table is missing");
        std::string err;
        g->ctc_shape = CheckCtcShape(*g->host_plan, &err) ? 0 : 1;
        g->ctc_shape_err = err;
    }
    if (g->ctc_shape != 0) return Fail("ctc_beam_search(crf=1): " + g->ctc_shape_err);
    if (g->out_off) return 0;
    const DenPlan &h = *g->host_plan;
    int *off = nullptr, *dst = nullptr;
    float *w = nullptr;
    if (Upload(&off, h.out_off) || Upload(&dst, h.out_dst) || Upload(&w, h.out_w)) {
        cudaFree(off); cudaFree(dst); cudaFree(w);
        return 1;
    }
    g->out_dst = dst; g->out_w = w; g->out_off = off;
    return 0;
}

size_t ccb_ctc_beam_search_ws_bytes(int N, int T, int beam) {
    return N > 0 && T > 0 && beam >= 1 && beam <= kBeamMax ? BeamWsBytes(N, T, beam) : 0;
}

int ccb_ctc_beam_search(const void *logits, int dtype, int N, int T, int V, const int *len_dev, int beam, int cutoff_top_n,
                        int crf, void *workspace, int *tokens, int *lengths, int *timesteps, float *scores, void *stream) {
    return ccb_ctc_beam_search_lm(logits, dtype, N, T, V, len_dev, beam, cutoff_top_n, crf, workspace, tokens, lengths,
                                  timesteps, scores, nullptr, 0.0, 0.0, stream);
}

int ccb_ctc_beam_search_lm(const void *logits, int dtype, int N, int T, int V, const int *len_dev, int beam, int cutoff_top_n,
                           int crf, void *workspace, int *tokens, int *lengths, int *timesteps, float *scores, const void *lm,
                           double alpha, double beta, void *stream) {
    g_err.clear();
    if (N <= 0 || T <= 0 || V <= 0) return Fail("ctc_beam_search: N, T and V must be positive");
    if (!KnownDtype(dtype)) return FailDtype("ctc_beam_search", dtype);
    if (beam < 1 || beam > kBeamMax)
        return Fail("ctc_beam_search: beam must lie in [1, " + std::to_string(kBeamMax) + "], not " + std::to_string(beam));
    if (cutoff_top_n < 1 || cutoff_top_n > V)
        return Fail("ctc_beam_search: cutoff_top_n must lie in [1, V] = [1, " + std::to_string(V) + "], not " +
                    std::to_string(cutoff_top_n));
    if (V > kBeamMaxV) return Fail("ctc_beam_search: at most " + std::to_string(kBeamMaxV) + " labels, not " + std::to_string(V));
    if (!logits || !len_dev || !workspace || !tokens || !lengths || !timesteps || !scores)
        return Fail("ctc_beam_search: missing buffer");
    const NGramDev *lmd = nullptr;
    if (lm) {
        NGram *m = reinterpret_cast<NGram *>(const_cast<void *>(lm));
        if (crf) return Fail("ctc_beam_search: an n-gram LM cannot be combined with crf=1 (the den graph has its own LM)");
        if (!(std::isfinite(alpha) && alpha >= 0.0)) return Fail("ctc_beam_search: alpha must be finite and >= 0");
        if (!std::isfinite(beta)) return Fail("ctc_beam_search: beta must be finite");
        if (m->host.V != V)
            return Fail("ctc_beam_search: the LM was loaded for " + std::to_string(m->host.V) + " labels, V is " + std::to_string(V));
        if (EnsureNGram(m, &lmd)) return 1;
    }
    DeviceGraph *g = nullptr;
    if (crf) {
        if (CurrentGraph(&g)) return 1;
        if (g->num_labels > V)
            return Fail("ctc_beam_search: the den graph has labels up to " + std::to_string(g->num_labels - 1) + ", V is " +
                        std::to_string(V));
        if (EnsureBeamGraph(g)) return 1;
    }
    const int rc = LaunchBeamSearch(g, logits, dtype, N, T, V, len_dev, beam, cutoff_top_n, workspace, tokens, lengths,
                                    timesteps, scores, (cudaStream_t)stream, lmd, alpha, beta);
    if (rc) return FailCuda("beam_search", (cudaError_t)rc);
    return 0;
}

/* ---- token n-gram LM ------------------------------------------------------------------------ */
void *ccb_ngram_create(const char *path, const char *const *labels, int V) {
    g_err.clear();
    NGram *m = new NGram();
    std::string err;
    if (!LoadArpa(path, labels, V, &m->host, &err)) { g_err = err; delete m; return nullptr; }
    return m;
}

void ccb_ngram_destroy(void *lm) {
    if (!lm) return;
    NGram *m = reinterpret_cast<NGram *>(lm);
    {
        std::lock_guard<std::mutex> lk(g_mu);
        int prev = -1;
        for (int d = 0; d < kMaxDevices; ++d) {
            if (!m->uploaded[d]) continue;
            if (prev < 0) cudaGetDevice(&prev);
            if (cudaSetDevice(d) != cudaSuccess) continue;
            for (void *p : m->blocks[d]) cudaFree(p);
        }
        if (prev >= 0) cudaSetDevice(prev);
    }
    delete m;
}

int ccb_ngram_info(void *lm, long *info) {
    if (!lm || !info) return 1;
    const NGramHost &h = reinterpret_cast<const NGram *>(lm)->host;
    const long v[] = {h.order, h.num_states(), h.num_arcs(), h.unk_substituted ? 1 : 0, h.W, h.V, h.bos, h.eos};
    memcpy(info, v, sizeof(v));
    for (int k = 0; k < kNgramMaxOrder; ++k) info[8 + k] = h.counts[k];
    return 0;
}

int ccb_ngram_copy(void *lm, int which, void *dst, size_t dst_bytes) {
    if (!lm || !dst) return 1;
    const NGramHost &h = reinterpret_cast<const NGram *>(lm)->host;
    const void *src = nullptr;
    size_t bytes = 0;
    switch (which) {
        case 0: src = h.tok2word.data(); bytes = h.tok2word.size() * 4; break;
        case 1: src = h.root_p.data(); bytes = h.root_p.size() * 4; break;
        case 2: src = h.root_dst.data(); bytes = h.root_dst.size() * 4; break;
        case 3: src = h.arc_off.data(); bytes = h.arc_off.size() * 4; break;
        case 4: src = h.arc_word.data(); bytes = h.arc_word.size() * 4; break;
        case 5: src = h.arc_p.data(); bytes = h.arc_p.size() * 4; break;
        case 6: src = h.arc_dst.data(); bytes = h.arc_dst.size() * 4; break;
        case 7: src = h.bow.data(); bytes = h.bow.size() * 4; break;
        case 8: src = h.back.data(); bytes = h.back.size() * 4; break;
        default: return 1;
    }
    if (bytes > dst_bytes) return 2;
    if (bytes) memcpy(dst, src, bytes);
    return 0;
}

int ccb_ngram_slot_rows(const void *lm, int N, int beam, int V, const int *parent, const int *token, const int *state_in,
                        int *state_out, float *rows, void *stream) {
    g_err.clear();
    if (!lm) return Fail("ngram_slot_rows: missing LM");
    NGram *m = reinterpret_cast<NGram *>(const_cast<void *>(lm));
    if (N <= 0 || V <= 0) return Fail("ngram_slot_rows: N and V must be positive");
    if (beam < 1 || beam > kBeamMax)
        return Fail("ngram_slot_rows: beam must lie in [1, " + std::to_string(kBeamMax) + "], not " + std::to_string(beam));
    if (m->host.V != V)
        return Fail("ngram_slot_rows: the LM was loaded for " + std::to_string(m->host.V) + " labels, V is " + std::to_string(V));
    if ((parent && (!token || !state_in)) || !state_out || !rows) return Fail("ngram_slot_rows: missing buffer");
    const size_t smem = NgramSlotRowsSmemBytes(m->host.W);
    if (smem > 200 * 1024)
        return Fail("ngram_slot_rows: the LM has " + std::to_string(m->host.W) + " words; its rows are built in shared "
                    "memory, which holds at most " + std::to_string(200 * 1024 / 8));
    const NGramDev *lmd = nullptr;
    if (EnsureNGram(m, &lmd)) return 1;
    const int rc = LaunchNgramSlotRows(*lmd, m->host.W, N, beam, V, parent, token, state_in, state_out, rows,
                                       (cudaStream_t)stream);
    if (rc) return FailCuda("ngram_slot_rows", (cudaError_t)rc);
    return 0;
}

int ccb_ngram_score(const void *lm, int R, int U, const void *ids, long ids_stride, int ids_i64, const void *last,
                    long last_stride, int last_i64, const void *lens, int lens_i64, float *out, void *stream) {
    g_err.clear();
    if (!lm) return Fail("ngram_score: missing LM");
    NGram *m = reinterpret_cast<NGram *>(const_cast<void *>(lm));
    if (R <= 0 || U <= 0) return Fail("ngram_score: R and U must be positive");
    if (ids_stride < U || last_stride < 0) return Fail("ngram_score: ids_stride must be >= U and last_stride >= 0");
    if ((ids_i64 | last_i64 | lens_i64) & ~1) return Fail("ngram_score: the *_i64 flags are 0 (int32) or 1 (int64)");
    if (!ids || !last || !out) return Fail("ngram_score: missing buffer");
    if (m->host.bos_word < 0 || !m->host.eos_listed)
        return Fail(std::string("ngram_score: the LM lists no ") + (m->host.bos_word < 0 ? "<s>" : "</s>") +
                    "; a sentence score starts with <s> and ends with </s>");
    const NGramDev *lmd = nullptr;
    if (EnsureNGram(m, &lmd)) return 1;
    NGramScoreArgs a;
    a.lm = *lmd;
    a.V = m->host.V; a.order = m->host.order; a.bos_word = m->host.bos_word; a.R = R; a.U = U;
    a.ids = ids; a.ids_stride = ids_stride; a.ids_i64 = ids_i64;
    a.last = last; a.last_stride = last_stride; a.last_i64 = last_i64;
    a.lens = lens; a.lens_i64 = lens_i64; a.out = out;
    const int rc = LaunchNgramScore(a, (cudaStream_t)stream);
    if (rc) return FailCuda("ngram_score", (cudaError_t)rc);
    return 0;
}

int ccb_lm_mix_slot_rows(int n_ngram, const void *const *ngrams, const double *ngram_w, const int *const *state_in,
                         int *const *state_out, int n_neural, const void *const *neural_rows, const int *neural_dtype,
                         const double *neural_w, const int *order, int N, int beam, int V, const int *parent,
                         const int *token, float *rows, void *stream) {
    g_err.clear();
    const int K = n_ngram + n_neural;
    if (n_ngram < 0 || n_neural < 0 || K < 1 || K > kLmMixMax)
        return Fail("lm_mix_slot_rows: a mix has 1 to " + std::to_string(kLmMixMax) + " members, not " + std::to_string(K));
    if (N <= 0 || V <= 0) return Fail("lm_mix_slot_rows: N and V must be positive");
    if (beam < 1 || beam > kBeamMax)
        return Fail("lm_mix_slot_rows: beam must lie in [1, " + std::to_string(kBeamMax) + "], not " + std::to_string(beam));
    if (!order || (parent && !token) || !rows || (n_ngram && (!ngrams || !ngram_w || !state_out || (parent && !state_in))) ||
        (n_neural && (!neural_rows || !neural_dtype || !neural_w)))
        return Fail("lm_mix_slot_rows: missing buffer");
    LmMixDev mix;
    mix.K = K;
    bool seen[kLmMixMax] = {};
    int W = 0;
    for (int i = 0; i < K; ++i) {
        const int j = order[i];
        if (j < 0 || j >= K || seen[j])
            return Fail("lm_mix_slot_rows: order must be a permutation of the members 0 .. " + std::to_string(K - 1));
        seen[j] = true;
        LmMixMember &m = mix.m[i];
        if (j < n_ngram) {
            if (!ngrams[j]) return Fail("lm_mix_slot_rows: missing LM");
            if (!state_out[j] || (parent && !state_in[j])) return Fail("lm_mix_slot_rows: missing buffer");
            NGram *g = reinterpret_cast<NGram *>(const_cast<void *>(ngrams[j]));
            if (g->host.V != V)
                return Fail("lm_mix_slot_rows: an LM was loaded for " + std::to_string(g->host.V) + " labels, V is " +
                            std::to_string(V));
            m.w = ngram_w[j];
            m.W = g->host.W;
            m.state_in = parent ? state_in[j] : nullptr;
            m.state_out = state_out[j];
            W = std::max(W, m.W);
        } else {
            const int k = j - n_ngram;
            if (!neural_rows[k]) return Fail("lm_mix_slot_rows: missing buffer");
            if (!KnownDtype(neural_dtype[k])) return FailDtype("lm_mix_slot_rows", neural_dtype[k]);
            m.rows = neural_rows[k];
            m.dtype = neural_dtype[k];
            m.w = neural_w[k];
        }
        if (!std::isfinite(m.w) || m.w == 0.0) return Fail("lm_mix_slot_rows: the weights must be finite and non-zero");
    }
    if (LmMixSlotRowsSmemBytes(W, V) > 200 * 1024)
        return Fail("lm_mix_slot_rows: the largest LM has " + std::to_string(W) + " words and V is " + std::to_string(V) +
                    "; the rows are built in shared memory, which holds at most " + std::to_string(200 * 1024 / 8) +
                    " words plus labels");
    for (int i = 0; i < K; ++i) {   // the n-gram tables on the device (uploaded once per LM and device)
        if (mix.m[i].rows) continue;
        const NGramDev *lmd = nullptr;
        if (EnsureNGram(reinterpret_cast<NGram *>(const_cast<void *>(ngrams[order[i]])), &lmd)) return 1;
        mix.m[i].lm = *lmd;
    }
    const int rc = LaunchLmMixSlotRows(mix, W, N, beam, V, parent, token, rows, (cudaStream_t)stream);
    if (rc) return FailCuda("lm_mix_slot_rows", (cudaError_t)rc);
    return 0;
}

/* ---- TLG decoding graph and its Viterbi beam search ------------------------------------------- */
// A decoding graph handle (ccb_wfst_create): the host tables, and their device copies, uploaded by the first search that
// uses the graph on a device and freed by ccb_wfst_destroy
struct Wfst {
    WfstHost host;
    bool uploaded[kMaxDevices] = {};
    WfstDev dev[kMaxDevices];
    std::vector<void *> blocks[kMaxDevices];
};

static WfstDev WfstShape(const WfstHost &h) {
    WfstDev t;
    t.S = h.S; t.start = h.start; t.L = h.L; t.E = h.E; t.max_out = h.max_out;
    return t;
}

static int EnsureWfst(Wfst *m, const WfstDev **out) {
    std::lock_guard<std::mutex> lk(g_mu);
    int d = 0;
    CCB_CUDA(cudaGetDevice(&d));
    if (d < 0 || d >= kMaxDevices) return Fail("wfst_decode: CUDA device " + std::to_string(d) + " is out of range");
    if (!m->uploaded[d]) {
        const WfstHost &h = m->host;
        WfstDev t = WfstShape(h);
        int *arc_off = nullptr, *eps_off = nullptr, *dst = nullptr, *tok = nullptr, *olabel = nullptr, *fid = nullptr,
            *src = nullptr, *lay = nullptr, *level = nullptr;
        float *w = nullptr, *fin = nullptr;
        const int rc = Upload(&arc_off, h.arc_off) || Upload(&eps_off, h.eps_off) || Upload(&dst, h.dst) ||
                       Upload(&tok, h.tok) || Upload(&olabel, h.olabel) || Upload(&fid, h.fid) || Upload(&src, h.src) ||
                       Upload(&lay, h.lay) || Upload(&level, h.level) || Upload(&w, h.w) || Upload(&fin, h.final_cost);
        m->blocks[d] = {arc_off, eps_off, dst, tok, olabel, fid, src, lay, level, w, fin};
        if (rc) {
            for (void *p : m->blocks[d]) cudaFree(p);
            m->blocks[d].clear();
            return 1;
        }
        t.arc_off = arc_off; t.eps_off = eps_off; t.dst = dst; t.tok = tok; t.olabel = olabel; t.fid = fid; t.src = src;
        t.lay = lay; t.level = level; t.w = w; t.final_cost = fin;
        m->dev[d] = t;
        m->uploaded[d] = true;
    }
    *out = &m->dev[d];
    return 0;
}

void *ccb_wfst_create(const char *path) {
    g_err.clear();
    Wfst *m = new Wfst();
    std::string err;
    if (!LoadWfst(path, &m->host, &err)) { g_err = err; delete m; return nullptr; }
    return m;
}

void ccb_wfst_destroy(void *graph) {
    if (!graph) return;
    Wfst *m = reinterpret_cast<Wfst *>(graph);
    {
        std::lock_guard<std::mutex> lk(g_mu);
        int prev = -1;
        for (int d = 0; d < kMaxDevices; ++d) {
            if (!m->uploaded[d]) continue;
            if (prev < 0) cudaGetDevice(&prev);
            if (cudaSetDevice(d) != cudaSuccess) continue;
            for (void *p : m->blocks[d]) cudaFree(p);
        }
        if (prev >= 0) cudaSetDevice(prev);
    }
    delete m;
}

int ccb_wfst_info(void *graph, long *info) {
    if (!graph || !info) return 1;
    const WfstHost &h = reinterpret_cast<const Wfst *>(graph)->host;
    const long v[] = {h.S, h.A, h.start, h.L, h.E, h.max_out, h.max_ilabel, h.eps_arcs};
    memcpy(info, v, sizeof(v));
    return 0;
}

int ccb_wfst_copy(void *graph, int which, void *dst, size_t dst_bytes) {
    if (!graph || !dst) return 1;
    const WfstHost &h = reinterpret_cast<const Wfst *>(graph)->host;
    const void *src = nullptr;
    size_t bytes = 0;
    switch (which) {
        case 0: src = h.arc_off.data(); bytes = h.arc_off.size() * 4; break;
        case 1: src = h.eps_off.data(); bytes = h.eps_off.size() * 4; break;
        case 2: src = h.dst.data(); bytes = h.dst.size() * 4; break;
        case 3: src = h.tok.data(); bytes = h.tok.size() * 4; break;
        case 4: src = h.olabel.data(); bytes = h.olabel.size() * 4; break;
        case 5: src = h.w.data(); bytes = h.w.size() * 4; break;
        case 6: src = h.fid.data(); bytes = h.fid.size() * 4; break;
        case 7: src = h.final_cost.data(); bytes = h.final_cost.size() * 4; break;
        case 8: src = h.level.data(); bytes = h.level.size() * 4; break;
        default: return 1;
    }
    if (bytes > dst_bytes) return 2;
    if (bytes) memcpy(dst, src, bytes);
    return 0;
}

size_t ccb_wfst_decode_ws_bytes(void *graph, int N, int T, int max_active) {
    if (!graph || N <= 0 || T <= 0 || max_active < 1 || max_active > kWfstMaxActive) return 0;
    return WfstWsBytes(WfstShape(reinterpret_cast<const Wfst *>(graph)->host), N, T, max_active);
}

int ccb_wfst_decode(const void *logits, int dtype, int N, int T, int V, const int *len_dev, void *graph, float acwt,
                    float lmwt, float wip, float beam, int max_active, void *workspace, int *words, int *num_words,
                    int *align, float *ac_logp, float *graph_cost, float *cost, int *reached_final, void *stream) {
    g_err.clear();
    if (!graph) return Fail("wfst_decode: null graph");
    if (N <= 0 || T <= 0 || V <= 0) return Fail("wfst_decode: N, T and V must be positive");
    if (!KnownDtype(dtype)) return FailDtype("wfst_decode", dtype);
    if (V > kWfstMaxV) return Fail("wfst_decode: at most " + std::to_string(kWfstMaxV) + " labels, not " + std::to_string(V));
    if (max_active < 1 || max_active > kWfstMaxActive)
        return Fail("wfst_decode: max_active must lie in [1, " + std::to_string(kWfstMaxActive) + "], not " +
                    std::to_string(max_active));
    if (!(beam > 0.f)) return Fail("wfst_decode: beam must be > 0 (inf is allowed)");
    if (!(std::isfinite(acwt) && acwt >= 0.f)) return Fail("wfst_decode: acwt must be finite and >= 0");
    if (!(std::isfinite(lmwt) && lmwt > 0.f)) return Fail("wfst_decode: lmwt must be finite and > 0");
    if (!std::isfinite(wip)) return Fail("wfst_decode: wip must be finite");
    Wfst *m = reinterpret_cast<Wfst *>(graph);
    if (m->host.max_ilabel > V)
        return Fail("wfst_decode: the graph has ilabels up to " + std::to_string(m->host.max_ilabel) + " (tokens up to " +
                    std::to_string(m->host.max_ilabel - 1) + "), V is " + std::to_string(V));
    if (!logits || !len_dev || !workspace || !words || !num_words || !align || !ac_logp || !graph_cost || !cost || !reached_final)
        return Fail("wfst_decode: missing buffer");
    const WfstDev *g = nullptr;
    if (EnsureWfst(m, &g)) return 1;
    const int rc = LaunchWfstDecode(*g, logits, dtype, N, T, V, len_dev, acwt, lmwt, wip, beam, max_active, workspace, words,
                                    num_words, align, ac_logp, graph_cost, cost, reached_final, (cudaStream_t)stream);
    if (rc) return FailCuda("wfst_decode", (cudaError_t)rc);
    return 0;
}

size_t ccb_rnnt_workspace_bytes(int N, long rows) { return N > 0 && rows >= 0 ? TransducerLoss<false>::WsBytes(N, rows) : 0; }

int ccb_rnnt_forward(const void *x, int dtype, int from_logits, int compact, int N, long rows, int V, int Tmax, int Umax,
                     const int *labels_dev, long n_labels, const int *lx_dev, const int *ly_dev, int blank, int want_beta,
                     void *workspace, float *costs, float *costs_beta, void *stream) {
    return TransducerForward<false>("rnnt_forward", x, dtype, from_logits, compact, N, rows, V, Tmax, Umax, labels_dev, n_labels,
                                    lx_dev, ly_dev, blank, want_beta, workspace, costs, costs_beta, stream);
}

int ccb_rnnt_backward(const void *x, int dtype, int from_logits, int N, long rows, int V, const int *labels_dev, int blank,
                      void *workspace, const float *w, void *grad, void *stream) {
    return TransducerBackward<false>("rnnt_backward", x, dtype, from_logits, N, rows, V, labels_dev, blank, workspace, w, grad,
                                     stream);
}

size_t ccb_rnnt_simple_workspace_bytes(int N, int Tmax, int Umax) {
    return N > 0 && Tmax > 0 && Umax >= 0 ? TransducerLoss<false>::SimpleWsBytes(N, Tmax, Umax) : 0;
}

int ccb_rnnt_simple_forward(const void *f, const void *g, int dtype, int N, int Tmax, int Umax, int V, const int *labels_dev,
                            const int *lx_dev, const int *ly_dev, int blank, int want_beta, void *workspace, float *costs,
                            void *stream) {
    return SimpleForward<false>("rnnt_simple_forward", f, g, dtype, N, Tmax, Umax, V, labels_dev, lx_dev, ly_dev, blank,
                                want_beta, workspace, costs, stream);
}

int ccb_rnnt_simple_backward(const void *f, const void *g, int dtype, int N, int Tmax, int Umax, int V, const int *labels_dev,
                             int blank, void *workspace, const float *w, void *grad_f, void *grad_g, void *stream) {
    return SimpleBackward<false>("rnnt_simple_backward", f, g, dtype, N, Tmax, Umax, V, labels_dev, blank, workspace, w, grad_f,
                                 grad_g, stream);
}

size_t ccb_ctct_workspace_bytes(int N, long rows) { return N > 0 && rows >= 0 ? TransducerLoss<true>::WsBytes(N, rows) : 0; }

int ccb_ctct_forward(const void *x, int dtype, int from_logits, int compact, int N, long rows, int V, int Tmax, int Umax,
                     const int *labels_dev, long n_labels, const int *lx_dev, const int *ly_dev, int blank, int want_beta,
                     void *workspace, float *costs, float *costs_beta, void *stream) {
    return TransducerForward<true>("ctct_forward", x, dtype, from_logits, compact, N, rows, V, Tmax, Umax, labels_dev, n_labels,
                                   lx_dev, ly_dev, blank, want_beta, workspace, costs, costs_beta, stream);
}

int ccb_ctct_backward(const void *x, int dtype, int from_logits, int N, long rows, int V, const int *labels_dev, int blank,
                      void *workspace, const float *w, void *grad, void *stream) {
    return TransducerBackward<true>("ctct_backward", x, dtype, from_logits, N, rows, V, labels_dev, blank, workspace, w, grad,
                                    stream);
}

size_t ccb_ctct_simple_workspace_bytes(int N, int Tmax, int Umax) {
    return N > 0 && Tmax > 0 && Umax >= 0 ? TransducerLoss<true>::SimpleWsBytes(N, Tmax, Umax) : 0;
}

int ccb_ctct_simple_forward(const void *f, const void *g, int dtype, int N, int Tmax, int Umax, int V, const int *labels_dev,
                            const int *lx_dev, const int *ly_dev, int blank, int want_beta, void *workspace, float *costs,
                            void *stream) {
    return SimpleForward<true>("ctct_simple_forward", f, g, dtype, N, Tmax, Umax, V, labels_dev, lx_dev, ly_dev, blank,
                               want_beta, workspace, costs, stream);
}

int ccb_ctct_simple_backward(const void *f, const void *g, int dtype, int N, int Tmax, int Umax, int V, const int *labels_dev,
                             int blank, void *workspace, const float *w, void *grad_f, void *grad_g, void *stream) {
    return SimpleBackward<true>("ctct_simple_backward", f, g, dtype, N, Tmax, Umax, V, labels_dev, blank, workspace, w, grad_f,
                                grad_g, stream);
}

/* ---- transducer beam search ------------------------------------------------------------------ */
static int CheckRnntBeam(const char *what, int N, int Tmax, int beam) {
    if (N <= 0 || Tmax < 0) return Fail(std::string(what) + ": N must be positive and Tmax >= 0");
    if (beam < 1 || beam > kBeamMax)
        return Fail(std::string(what) + ": beam must lie in [1, " + std::to_string(kBeamMax) + "], not " + std::to_string(beam));
    return 0;
}

size_t ccb_rnnt_beam_ws_bytes(int N, int Tmax, int beam) {
    return N > 0 && Tmax >= 0 && beam >= 1 && beam <= kBeamMax ? RnntBeamWsBytes(N, Tmax, beam) : 0;
}

int ccb_rnnt_beam_init(int N, int Tmax, int beam, void *workspace, int *parent, int *token, int *node, double *score,
                       void *stream) {
    g_err.clear();
    if (CheckRnntBeam("rnnt_beam_init", N, Tmax, beam)) return 1;
    if (!workspace || !parent || !token || !node || !score) return Fail("rnnt_beam_init: missing buffer");
    const int rc = LaunchRnntBeamInit(N, Tmax, beam, workspace, parent, token, node, score, (cudaStream_t)stream);
    if (rc) return FailCuda("rnnt_beam_init", (cudaError_t)rc);
    return 0;
}

// the arguments every transducer step entry takes (RNN-T and CTC-T)
static int CheckRnntStep(const char *what, const void *rows, const void *enc, int dtype, int mode, int N, int Tmax, int beam,
                         int V, int t, const int *len_dev, int blank, void *workspace, int *parent, int *token, int *node,
                         double *score) {
    const std::string w(what);
    if (CheckRnntBeam(what, N, Tmax, beam)) return 1;
    if (!KnownDtype(dtype)) return FailDtype(what, dtype);
    if (mode < 0 || mode > 2) return Fail(w + ": mode must be 0 (log-probs), 1 (logits) or 2 (LogAdd)");
    if (V <= 0 || V > kRnntBeamMaxV) return Fail(w + ": V must lie in [1, 2^24], not " + std::to_string(V));
    if (t < 0 || t >= Tmax) return Fail(w + ": frame t must lie in [0, Tmax)");
    if (blank < 0 || blank >= V) return Fail(w + ": blank must lie in [0, V)");
    if (!rows || (mode == 2 && !enc) || !len_dev || !workspace || !parent || !token || !node || !score)
        return Fail(w + ": missing buffer");
    return 0;
}

int ccb_rnnt_beam_step(const void *rows, const void *enc, int dtype, int mode, int N, int Tmax, int beam, int V, int t,
                       const int *len_dev, int blank, void *workspace, int *parent, int *token, int *node, double *score,
                       void *stream) {
    g_err.clear();
    if (CheckRnntStep("rnnt_beam_step", rows, enc, dtype, mode, N, Tmax, beam, V, t, len_dev, blank, workspace, parent, token,
                      node, score))
        return 1;
    const int rc = LaunchRnntBeamStep(rows, enc, dtype, mode, N, Tmax, beam, V, t, len_dev, blank, workspace, parent, token,
                                      node, score, (cudaStream_t)stream);
    if (rc) return FailCuda("rnnt_beam_step", (cudaError_t)rc);
    return 0;
}

int ccb_rnnt_beam_step_fused(const void *rows, const void *enc, int dtype, int mode, int N, int Tmax, int beam, int V, int t,
                             const int *len_dev, int blank, void *workspace, int *parent, int *token, int *node,
                             double *score, const void *lm_rows, int lm_dtype, double alpha, double beta,
                             const void *ilm_rows, int ilm_dtype, double ilm_weight, double *lm_part, void *stream) {
    g_err.clear();
    if (CheckRnntStep("rnnt_beam_step_fused", rows, enc, dtype, mode, N, Tmax, beam, V, t, len_dev, blank, workspace, parent,
                      token, node, score))
        return 1;
    if (!lm_rows && !ilm_rows)
        return Fail("rnnt_beam_step_fused: neither LM rows nor ILM rows: use rnnt_beam_step for the search without fusion");
    if (!lm_part) return Fail("rnnt_beam_step_fused: missing buffer");
    if (lm_rows && !KnownDtype(lm_dtype)) return FailDtype("rnnt_beam_step_fused", lm_dtype);
    if (ilm_rows && !KnownDtype(ilm_dtype)) return FailDtype("rnnt_beam_step_fused", ilm_dtype);
    if (!std::isfinite(alpha) || !std::isfinite(beta) || !std::isfinite(ilm_weight))
        return Fail("rnnt_beam_step_fused: alpha, beta and ilm_weight must be finite");
    const int rc = LaunchRnntBeamStepFused(rows, enc, dtype, mode, N, Tmax, beam, V, t, len_dev, blank, workspace, parent,
                                           token, node, score, lm_rows, lm_dtype, alpha, beta, ilm_rows, ilm_dtype,
                                           ilm_weight, lm_part, (cudaStream_t)stream);
    if (rc) return FailCuda("rnnt_beam_step_fused", (cudaError_t)rc);
    return 0;
}

int ccb_rnnt_beam_finish(int N, int Tmax, int beam, int nbest, const void *workspace, const int *node, const double *score,
                         int *tokens, int *lengths, float *scores, void *stream) {
    g_err.clear();
    if (CheckRnntBeam("rnnt_beam_finish", N, Tmax, beam)) return 1;
    if (nbest < 1 || nbest > beam) return Fail("rnnt_beam_finish: nbest must lie in [1, beam]");
    if (!workspace || !node || !score || (Tmax && !tokens) || !lengths || !scores) return Fail("rnnt_beam_finish: missing buffer");
    const int rc = LaunchRnntBeamFinish(N, Tmax, beam, nbest, workspace, node, score, tokens, lengths, scores,
                                        (cudaStream_t)stream);
    if (rc) return FailCuda("rnnt_beam_finish", (cudaError_t)rc);
    return 0;
}

/* ---- CTC-T beam search (finished by ccb_rnnt_beam_finish) ------------------------------------- */
size_t ccb_ctct_beam_ws_bytes(int N, int Tmax, int beam) {
    return N > 0 && Tmax >= 0 && beam >= 1 && beam <= kBeamMax ? CtctBeamWsBytes(N, Tmax, beam) : 0;
}

int ccb_ctct_beam_init(int N, int Tmax, int beam, void *workspace, int *parent, int *token, int *node, double *score,
                       void *stream) {
    g_err.clear();
    if (CheckRnntBeam("ctct_beam_init", N, Tmax, beam)) return 1;
    if (!workspace || !parent || !token || !node || !score) return Fail("ctct_beam_init: missing buffer");
    const int rc = LaunchCtctBeamInit(N, Tmax, beam, workspace, parent, token, node, score, (cudaStream_t)stream);
    if (rc) return FailCuda("ctct_beam_init", (cudaError_t)rc);
    return 0;
}

int ccb_ctct_beam_step(const void *rows, const void *enc, int dtype, int mode, int N, int Tmax, int beam, int V, int t,
                       const int *len_dev, int blank, void *workspace, int *parent, int *token, int *node, double *score,
                       void *stream) {
    g_err.clear();
    if (CheckRnntStep("ctct_beam_step", rows, enc, dtype, mode, N, Tmax, beam, V, t, len_dev, blank, workspace, parent, token,
                      node, score))
        return 1;
    const int rc = LaunchCtctBeamStep(rows, enc, dtype, mode, N, Tmax, beam, V, t, len_dev, blank, workspace, parent, token,
                                      node, score, (cudaStream_t)stream);
    if (rc) return FailCuda("ctct_beam_step", (cudaError_t)rc);
    return 0;
}

size_t ccb_gather_ws_bytes(int N) { return N > 0 ? GatherWsBytes(N) : 0; }

int ccb_gather_sum(const void *a, const void *b, int dtype, int N, long rows_out, int H, const int *la_dev, const int *lb_dev,
                   void *workspace, void *out, void *stream) {
    g_err.clear();
    if (N <= 0 || rows_out < 0 || H <= 0) return Fail("gather_sum: N and H must be positive, rows_out >= 0");
    if (!KnownDtype(dtype)) return FailDtype("gather_sum", dtype);
    if (!a || !b || !la_dev || !lb_dev || !workspace || (rows_out && !out)) return Fail("gather_sum: missing buffer");
    const int rc = LaunchGatherSum(a, b, dtype, N, rows_out, H, la_dev, lb_dev, workspace, out, (cudaStream_t)stream);
    if (rc) return FailCuda("gather_sum", (cudaError_t)rc);
    return 0;
}

int ccb_gather_sum_backward(const void *grad_out, int dtype, int N, long rows_a, long rows_b, int H, const int *la_dev,
                            const int *lb_dev, void *workspace, void *grad_a, void *grad_b, void *stream) {
    g_err.clear();
    if (N <= 0 || rows_a < 0 || rows_b < 0 || H <= 0) return Fail("gather_sum_backward: N and H must be positive");
    if (!KnownDtype(dtype)) return FailDtype("gather_sum_backward", dtype);
    if (!grad_out || !la_dev || !lb_dev || !workspace || !grad_a || !grad_b) return Fail("gather_sum_backward: missing buffer");
    const int rc = LaunchGatherSumBackward(grad_out, dtype, N, rows_a, rows_b, H, la_dev, lb_dev, workspace, grad_a, grad_b,
                                           (cudaStream_t)stream);
    if (rc) return FailCuda("gather_sum_backward", (cudaError_t)rc);
    return 0;
}

/* ---- gpu_ctc/ctc.h surface ------------------------------------------------------------------- */
const char *ctcGetStatusString(ctcStatus_t status) {
    switch (status) {
        case CTC_STATUS_SUCCESS: return "no error";
        case CTC_STATUS_MEMOPS_FAILED: return "cuda memcpy or memset failed";
        case CTC_STATUS_INVALID_VALUE: return "invalid value";
        case CTC_STATUS_EXECUTION_FAILED: return "execution failed";
        default: return "unknown error";
    }
}

// workspace: [meta ints: labels | label_off | label_len | len] then the alpha spill
ctcStatus_t get_workspace_size(const int *const label_lengths, const int *const input_lengths, int alphabet_size,
                               int minibatch, struct ctcOptions options, size_t *size_bytes) {
    (void)options;
    if (!label_lengths || !input_lengths || !size_bytes || alphabet_size <= 0 || minibatch <= 0) return CTC_STATUS_INVALID_VALUE;
    int maxL = 0, maxT = 0;
    long sumL = 0;
    for (int i = 0; i < minibatch; ++i) {
        if (label_lengths[i] < 0 || input_lengths[i] < 0) return CTC_STATUS_INVALID_VALUE;
        maxL = std::max(maxL, label_lengths[i]); maxT = std::max(maxT, input_lengths[i]); sumL += label_lengths[i];
    }
    size_t meta = ((size_t)(sumL + 3 * (size_t)minibatch + 1) * sizeof(int) + 255) & ~(size_t)255;
    *size_bytes = meta + ((size_t)minibatch * sizeof(float) + 255 & ~(size_t)255) + ccb_ctc_workspace_bytes(minibatch, maxT, maxL);
    return CTC_STATUS_SUCCESS;
}

ctcStatus_t compute_ctc_loss(const float *const activations, float *gradients, const int *const flat_labels,
                             const int *const label_lengths, const int *const input_lengths, int alphabet_size,
                             int minibatch, float *costs, void *workspace, struct ctcOptions options) {
    if (!activations || !flat_labels || !label_lengths || !input_lengths || !costs || !workspace || alphabet_size <= 0 || minibatch <= 0)
        return CTC_STATUS_INVALID_VALUE;
    int maxL = 0, maxT = 0;
    std::vector<int> meta;
    long sumL = 0;
    for (int i = 0; i < minibatch; ++i) { maxL = std::max(maxL, label_lengths[i]); maxT = std::max(maxT, input_lengths[i]); sumL += label_lengths[i]; }
    meta.reserve((size_t)sumL + 3 * (size_t)minibatch + 1);
    meta.insert(meta.end(), flat_labels, flat_labels + sumL);
    int off = 0;
    for (int i = 0; i < minibatch; ++i) { meta.push_back(off); off += label_lengths[i]; }
    meta.push_back(off);
    meta.insert(meta.end(), label_lengths, label_lengths + minibatch);
    meta.insert(meta.end(), input_lengths, input_lengths + minibatch);
    for (long i = 0; i < sumL; ++i) if (flat_labels[i] < 0 || flat_labels[i] >= alphabet_size) return CTC_STATUS_INVALID_VALUE;
    cudaStream_t s = (cudaStream_t)options.stream;
    char *ws = reinterpret_cast<char *>(workspace);
    const size_t meta_bytes = (meta.size() * sizeof(int) + 255) & ~(size_t)255;
    const size_t cost_bytes = ((size_t)minibatch * sizeof(float) + 255) & ~(size_t)255;
    if (cudaMemcpyAsync(ws, meta.data(), meta.size() * sizeof(int), cudaMemcpyHostToDevice, s) != cudaSuccess) return CTC_STATUS_MEMOPS_FAILED;
    // the host staging vector must outlive the (pageable => staged synchronously) copy: it does, pageable H2D
    // returns after the source has been consumed.
    const int *d_labels = reinterpret_cast<const int *>(ws);
    const int *d_off = d_labels + sumL;
    const int *d_llen = d_off + minibatch + 1;
    const int *d_len = d_llen + minibatch;
    float *d_costs = reinterpret_cast<float *>(ws + meta_bytes);
    float *alpha_ws = reinterpret_cast<float *>(ws + meta_bytes + cost_bytes);
    std::string err;
    // (T,N,V) layout: element (n,t,k) at t*(N*V) + n*V + k
    int rc = LaunchCtc(activations, 0, (long)alphabet_size, (long)minibatch * alphabet_size, minibatch, maxT, alphabet_size,
                       d_labels, d_off, d_llen, d_len, maxL, options.blank_label, alpha_ws, gradients,
                       (long)alphabet_size, (long)minibatch * alphabet_size, 1.f, d_costs, nullptr, s, &err);
    if (rc) { g_err = err; return CTC_STATUS_EXECUTION_FAILED; }
    if (cudaMemcpyAsync(costs, d_costs, sizeof(float) * minibatch, cudaMemcpyDeviceToHost, s) != cudaSuccess) return CTC_STATUS_MEMOPS_FAILED;
    if (cudaStreamSynchronize(s) != cudaSuccess) return CTC_STATUS_EXECUTION_FAILED;   // costs are host memory (gpu_ctc.h:365-368)
    return CTC_STATUS_SUCCESS;
}

/* ---- host-side plan inspection ------------------------------------------------------------------ */
void *ccb_plan_create(const char *fst_name, int n_ctas, int n_warps) {
    g_err.clear();
    HostFst fst;
    std::string err;
    if (!fst_name || !ReadFstFile(fst_name, &fst, &err)) { g_err = fst_name ? err : "null path"; return nullptr; }
    DenPlan *p = new DenPlan();
    if (!BuildDenPlan(fst, n_ctas, n_warps, p, &err)) { g_err = err; delete p; return nullptr; }
    return p;
}

void ccb_plan_destroy(void *plan) { delete reinterpret_cast<DenPlan *>(plan); }

int ccb_plan_info(void *plan, long *info) {
    if (!plan || !info) return 1;
    const DenPlan *p = reinterpret_cast<const DenPlan *>(plan);
    info[0] = p->file_states; info[1] = p->file_arcs; info[2] = p->num_states;
    info[3] = (long)p->fwd.arcs.size(); info[4] = (long)p->bwd.arcs.size(); info[5] = p->start;
    info[6] = p->num_labels; info[7] = p->n_ctas; info[8] = p->n_warps;
    info[9] = std::max(p->fwd.max_tile_arcs, p->bwd.max_tile_arcs);
    info[10] = p->num_pairs; info[11] = (long)p->start_arcs.size(); info[12] = (long)p->hub_states.size();
    return 0;
}

int ccb_plan_copy(void *plan, int which, void *dst, size_t dst_bytes) {
    if (!plan || !dst) return 1;
    const DenPlan *p = reinterpret_cast<const DenPlan *>(plan);
    const void *src = nullptr;
    size_t bytes = 0;
    switch (which) {
        case 0: src = p->state_label.data(); bytes = p->state_label.size() * 4; break;
        case 1: src = p->final_lin.data(); bytes = p->final_lin.size() * 4; break;
        case 2: src = p->orig_state.data(); bytes = p->orig_state.size() * 4; break;
        case 3: src = p->fwd.arcs.data(); bytes = p->fwd.arcs.size() * sizeof(Arc); break;
        case 4: src = p->fwd.chunk_state.data(); bytes = p->fwd.chunk_state.size() * 4; break;
        case 5: src = p->fwd.chunk_arc.data(); bytes = p->fwd.chunk_arc.size() * 4; break;
        case 6: src = p->bwd.arcs.data(); bytes = p->bwd.arcs.size() * sizeof(Arc); break;
        case 7: src = p->bwd.chunk_state.data(); bytes = p->bwd.chunk_state.size() * 4; break;
        case 8: src = p->bwd.chunk_arc.data(); bytes = p->bwd.chunk_arc.size() * 4; break;
        case 9: src = p->state_pos.data(); bytes = p->state_pos.size() * 4; break;
        case 10: src = p->fwd.chunk_pair.data(); bytes = p->fwd.chunk_pair.size() * 4; break;
        case 11: src = p->bwd.chunk_pair.data(); bytes = p->bwd.chunk_pair.size() * 4; break;
        case 12: src = p->start_arcs.data(); bytes = p->start_arcs.size() * sizeof(Arc); break;
        case 13: src = p->fwd.cta_labels.data(); bytes = p->fwd.cta_labels.size() * 4; break;
        case 14: src = p->bwd.cta_labels.data(); bytes = p->bwd.cta_labels.size() * 4; break;
        case 15: src = p->bwd.w1.data(); bytes = p->bwd.w1.size() * 4; break;
        case 16: src = p->hub_states.data(); bytes = p->hub_states.size() * 4; break;
        case 17: src = p->own_fwd.data(); bytes = (size_t)p->num_states * 2 * 4; break;   // (without the 4 floats of padding)
        case 18: src = p->own_bwd.data(); bytes = (size_t)p->num_states * 2 * 4; break;
        case 19: src = p->in_off.data(); bytes = p->in_off.size() * 4; break;
        case 20: src = p->in_src.data(); bytes = p->in_src.size() * 4; break;
        case 21: src = p->in_w.data(); bytes = p->in_w.size() * 4; break;
        case 22: src = p->out_off.data(); bytes = p->out_off.size() * 4; break;
        case 23: src = p->out_dst.data(); bytes = p->out_dst.size() * 4; break;
        case 24: src = p->out_w.data(); bytes = p->out_w.size() * 4; break;
        default: return 1;
    }
    if (bytes > dst_bytes) return 2;
    memcpy(dst, src, bytes);
    return 0;
}

int ccb_plan_ctc_shape(void *plan) {
    g_err.clear();
    if (!plan) return Fail("ccb_plan_ctc_shape: null plan");
    std::string err;
    return CheckCtcShape(*reinterpret_cast<const DenPlan *>(plan), &err) ? 0 : Fail(err);
}

static int PlanLaunch(void *plan, int N, int backward, int smem_optin, int hooks, DenLaunch *L, int *Npad) {
    const DenHooks h{(hooks & 1) != 0, (hooks & 2) != 0, (hooks & 4) != 0, (hooks & 8) != 0};
    const DenGraphShape g = ShapeOf(*reinterpret_cast<const DenPlan *>(plan), h);
    *Npad = PadLanes(N, SmallBatchOk(g, smem_optin, h));
    return ChooseDenLaunch(g, *Npad, backward != 0, smem_optin, h, L, &g_err) ? 0 : 1;
}

int ccb_plan_launch(void *plan, int N, int backward, int smem_optin, int hooks, long *out) {
    g_err.clear();
    if (!plan || !out || N <= 0) return Fail("ccb_plan_launch: bad arguments");
    DenLaunch L;
    int Npad = 0;
    if (PlanLaunch(plan, N, backward, smem_optin, hooks, &L, &Npad)) return 1;
    const long v[] = {L.tier, L.lanes_per_row, L.U, L.batch, L.w1_smem, Npad, L.tile_rows, L.gacc_rows, (long)L.arcs_off,
                      (long)L.ring_off, (long)L.bar_off, (long)L.w1_off, (long)L.abar_off, (long)L.aring_off, (long)L.total};
    memcpy(out, v, sizeof(v));
    return 0;
}

int ccb_plan_launch_own(void *plan, int N, int backward, int smem_optin, int hooks, long *out) {
    g_err.clear();
    if (!plan || !out || N <= 0) return Fail("ccb_plan_launch_own: bad arguments");
    DenLaunch L;
    int Npad = 0;
    if (PlanLaunch(plan, N, backward, smem_optin, hooks, &L, &Npad)) return 1;
    out[0] = L.own_smem;
    out[1] = (long)L.own_off;
    return 0;
}

}  // extern "C"
