// C ABI (include/siglip_b200.h) over the sm_90a kernels: context + workspaces, TMA descriptor encoding,
// the per-step chunk schedule, CUDA-IPC peer bootstrap. Host-side only; no torch types anywhere.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include <string>
#include <vector>

#include "../../include/siglip_b200.h"
#include "siglip_kernels.cuh"

using siglip::DebugRecord;
using siglip::KernelParams;
using siglip::Problem;

namespace {

thread_local std::string g_last_error;

int fail(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}

#define CK(call)                                                                                       \
  do {                                                                                                 \
    cudaError_t e__ = (call);                                                                          \
    if (e__ != cudaSuccess) {                                                                          \
      char buf__[512];                                                                                 \
      snprintf(buf__, sizeof(buf__), "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, \
               __LINE__);                                                                              \
      return fail(SIGLIP_ERR_CUDA, buf__);                                                             \
    }                                                                                                  \
  } while (0)

#define CKI(expr)                                                                                         \
  do {                                                                                                    \
    int e__ = (expr);                                                                                     \
    if (e__ != 0) {                                                                                       \
      char buf__[512];                                                                                    \
      snprintf(buf__, sizeof(buf__), "%s failed: %s (%s:%d)", #expr,                                      \
               cudaGetErrorString(static_cast<cudaError_t>(e__)), __FILE__, __LINE__);                    \
      return fail(SIGLIP_ERR_CUDA, buf__);                                                                \
    }                                                                                                     \
  } while (0)

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<EncodeTiledFn>(p);
    }
  }
  return fn;
}

// bf16 2-D tensor, `inner` contiguous elements per row, rows `row_stride_elems` apart; 128B-swizzled boxes.
int encode_bf16_2d(CUtensorMap* m, const void* base, uint64_t inner, uint64_t outer, uint64_t row_stride_elems,
                   uint32_t box_inner, uint32_t box_outer, CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return fail(SIGLIP_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  if ((reinterpret_cast<uintptr_t>(base) & 15u) != 0) return fail(SIGLIP_ERR_INVALID, "operand not 16-byte aligned");
  if ((row_stride_elems * 2) % 16 != 0) return fail(SIGLIP_ERR_INVALID, "row stride not a multiple of 16 bytes");
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {row_stride_elems * 2};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled failed with CUresult %d (inner=%llu outer=%llu stride=%llu)",
             static_cast<int>(r), (unsigned long long)inner, (unsigned long long)outer,
             (unsigned long long)row_stride_elems);
    return fail(SIGLIP_ERR_CUDA, buf);
  }
  return 0;
}

// 8-bit K-major operand [rows][K bytes]: 128-byte (= 128 element) swizzle rows
int encode_u8_kmajor(CUtensorMap* m, const void* base, int rows, int K, long long ld, int box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return fail(SIGLIP_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  if ((reinterpret_cast<uintptr_t>(base) & 15u) != 0 || (ld % 16) != 0)
    return fail(SIGLIP_ERR_INVALID, "8-bit operand needs a 16-byte aligned base and row stride");
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(K), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld)};
  cuuint32_t box[2] = {128, static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(SIGLIP_ERR_CUDA, "cuTensorMapEncodeTiled (uint8) failed");
  return 0;
}

// Operand tensor map for the mainloop. mn == 0: stored [rows][K], box {64 k, box_rows_kmajor rows};
// mn == 1: stored [K][rows], box {64 rows, box_k_mnmajor k}.
int encode_operand(CUtensorMap* m, const void* base, int rows, int K, long long ld, int mn, int box_rows_kmajor,
                   int box_k_mnmajor = 64) {
  if (!mn) return encode_bf16_2d(m, base, (uint64_t)K, (uint64_t)rows, (uint64_t)ld, 64, (uint32_t)box_rows_kmajor);
  return encode_bf16_2d(m, base, (uint64_t)rows, (uint64_t)K, (uint64_t)ld, 64, (uint32_t)box_k_mnmajor);
}

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
inline int round_up(int a, int b) { return ceil_div(a, b) * b; }

// The sigma operand G of the gradient contractions is stored as IEEE fp16 scaled by 2^14: 11 significant bits
// (bf16 has 8; its 2^-9 rounding was the whole 1e-3 error budget when negatives dominate a gradient), and every
// sigma down to 3.7e-9 (logit -19.4) stays a normal number. The out epilogue multiplies the accumulator by 2^-14.
constexpr float kGScale = 16384.0f;
// The embeddings enter the gradient contractions as fp16(x * 16): exact for every bf16 value with 3.8e-6 <= |x| <= 4094
// (L2-normalised embeddings live in [~1e-4, 1]); the conversion runs inside the loss kernel's idle warps.
constexpr float kXScale = 16.0f;
constexpr int kMaxWorld = 32;
// flags[kind][rank]: counters written by peers with st.release.sys
//   0 text of forward #n is in place        1 dtxt contribution of backward #n, gradient slot j is complete
//   2 forward #n finished pulling everyone's text     3 backward #n finished reading everyone's contributions
//   4 (dt', dbias) of backward #n are in the owner's mailbox (SIGLIP_OPT_SYNC_SCALAR_GRADS)
constexpr int kFlagKinds = 5;
// the mailbox (2 floats) lives behind the flag counters, in the same peer-mapped allocation
constexpr int kMailboxOffset = kFlagKinds * kMaxWorld;
constexpr size_t kFlagBytes = (kMailboxOffset + 4) * sizeof(unsigned int);
// local synchronisation words (zeroed at creation): one ticket per auxiliary-job position, the end-of-launch ticket,
// the "last fold complete" flag of the fused step
constexpr int kSyncEndTicket = siglip::kMaxAuxJobs;
constexpr int kSyncFoldDone = siglip::kMaxAuxJobs + 1;
constexpr int kSyncWords = 16;

struct IpcBlob {
  cudaIpcMemHandle_t txt;
  cudaIpcMemHandle_t slots;
  cudaIpcMemHandle_t flags;
  int rank;
  int device;
  int B;
  int D;
  int Bmax;
  char host[64];
};

}  // namespace

struct siglip_ctx {
  int device = 0, rank = 0, world = 1, B = 0, D = 0, Bp = 0;
  int Bs[kMaxWorld] = {};                // per-rank batch (all equal to B unless created with siglip_ctx_create_uneven)
  int Bmax = 0;                          // max over ranks: stride of every per-chunk buffer is Bmax * D elements
  int num_sms = 0;
  // options
  int cta_group = 2;
  int overlap_pull = 1;                  // pull the next text chunk inside the loss kernel
  int overlap_reduce = 1;                // fold the peers' dtxt contributions inside the gradient kernels
  int kernel_timing = 0;
  int stages_loss = 0, stages_grad = 0;  // 0 = kernel default
  int mcast = 1;                         // 2: vertically adjacent tiles share the B tile by TMA multicast
  int grad_bf16 = 0;                     // dimg / dtxt outputs are bf16 instead of fp32
  int sync_scalar_grads = 0;             // backward returns the mean over ranks of dt' / dbias
  int bidir = 0;                         // visiting order of the text chunks: r, r+1, r-1, r+2, r-2, ...
  int input_f16 = 0;                     // img / txt are fp16(x * kXScale) instead of bf16 (fp32-input path)
  int saved_f16 = 0;                     // format of the embeddings of the forward saved for backward
  int tprime_f64 = 0;                    // t_prime / dt_prime pointers of forward / backward / fwd_bwd are fp64 device scalars
  int pdl = 1;                           // programmatic dependent launch of the wgmma kernels (set-up overlaps the previous tail)
  int inkernel_sync = 1;                 // fused step: flags waited for / raised inside the wgmma kernels (0: helper launches)
  int split_k = 0;                       // gradient kernel: 0 = off (default), -1 = split a
                                         // ragged last wave automatically, S >= 2 = at most S slices
  long long peer_timeout_ms = 600000;    // bound of every wait on a peer (10 min: a peer may be saving a checkpoint)
  int aux_trace_on = 0;
  // diagnostics, read from the environment once at context creation (see include/siglip_b200.h)
  bool dbg_no_gstore = false, dbg_no_cvt = false, dbg_loss_waitstats = false;
  // workspaces
  __nv_bfloat16* txt_all = nullptr;      // [world][Bmax, D] bf16; slot `rank` is what the peers pull (world > 1)
  __nv_bfloat16* G[kMaxWorld] = {};      // [Bp, Bp] sigma operands (fp16 bits x kGScale), diagonal zeroed, allocated on
                                         // first use: fused step 2 (own chunk + the chunk in flight), split API one per chunk
  __nv_bfloat16* img16 = nullptr;        // [B, D] fp16 (x kXScale) images: B operand of the dtxt contraction
  __nv_bfloat16* txt16[kMaxWorld] = {};  // [Bmax, D] fp16 (x kXScale) text chunks: B operand of dimg (same count as G)
  float* g_diag = nullptr;               // [Bp] fp32 positive-pair terms -sigma(-z_ii)
  float* slots = nullptr;                // [world][Bmax, D] fp32 dtxt contributions, slot c is for owner c (world > 1)
  float* dimg_acc = nullptr;             // [B, D] fp32 running dimg over the chunks (world > 1)
  float* dtxt_acc = nullptr;             // [B, D] fp32 running sum of the peers' contributions (world > 1)
  double* partials = nullptr;            // [num_sms][4]
  unsigned int* fin_counter = nullptr;   // ticket counter of the loss kernel's last-CTA finalisation
  unsigned int* flags = nullptr;         // [kFlagKinds][kMaxWorld]
  unsigned int* sync_words = nullptr;    // [kSyncWords] local tickets / flags
  float* loop_mailboxes = nullptr;       // loopback only: [world][2] stand-ins for the peers' (dt', dbias) mailboxes
  float* loop_zero = nullptr;            // loopback only: [world][Bmax, D] zeros standing in for the peers' contribution slots
  float* scalars = nullptr;              // [24] device scalars: host API staging, saved dt'/dbias of the last forward
  unsigned long long* aux_trace = nullptr;  // [kTraceLaunches][16] globaltimer stamps (SIGLIP_OPT_AUX_TRACE)
  float* splitk_ws = nullptr;            // fp32 partial accumulators of the split tiles of the gradient kernel
  unsigned int* splitk_counters = nullptr;  // per split tile: arrivals of the non-owner parts (monotonic)
  size_t splitk_ws_bytes = 0;
  unsigned int aux_trace_n = 0;
  // peers (index = rank); own entries point at local memory
  __nv_bfloat16* peer_txt[kMaxWorld] = {};
  float* peer_slots[kMaxWorld] = {};
  unsigned int* peer_flags[kMaxWorld] = {};
  bool peers_ready = false;
  bool loopback = false;
  const float** reduce_ptrs_dev = nullptr;   // [world] peer_slots[p] + rank*stride  (reduction-at-the-end variant)
  const float** final_ptrs_dev = nullptr;    // [2] {dtxt_acc, own slot}: the local last add of the split API
  unsigned int** signal_ptrs_dev = nullptr;  // [kFlagKinds][world]
  const float** mailbox_ptrs_dev = nullptr;  // [world] every rank's (dt', dbias) mailbox
  unsigned int n_fwd = 0, n_bwd = 0;         // forward / backward passes issued (flag counters)
  unsigned int prewait3 = 0;                 // highest n for which "peers finished backward n" has been waited for
  unsigned long long gen = 0;                // generation of the state saved for backward (0 = none)
  DebugRecord* dbg_host = nullptr;
  DebugRecord* dbg_dev = nullptr;
  unsigned long long launches = 0;
  size_t workspace_bytes = 0;
  std::vector<cudaEvent_t> ev_loss, ev_grad;  // start, stop, start, stop, ...
  size_t ev_loss_used = 0, ev_grad_used = 0;
  // host-API staging
  __nv_bfloat16* h_img[2] = {nullptr, nullptr};   // device staging of the host entries, two sets (pipelining)
  __nv_bfloat16* h_txt[2] = {nullptr, nullptr};
  float* h_dimg = nullptr;
  float* h_dtxt = nullptr;
  __nv_bfloat16* h_gimg[2] = {nullptr, nullptr};  // bf16 gradient staging of the host entries that return gradients
  __nv_bfloat16* h_gtxt[2] = {nullptr, nullptr};
  float* h_pinned = nullptr;                       // pinned host: [2][8] = {t', bias, -, -, loss, dt', dbias, -} per set
  cudaStream_t copy_stream = nullptr, d2h_stream = nullptr;
  cudaEvent_t ev_h2d[2] = {nullptr, nullptr}, ev_step[2] = {nullptr, nullptr}, ev_done[2] = {nullptr, nullptr};
  unsigned long long host_submitted = 0;           // tickets handed out so far
};

namespace {

constexpr int kSavedScalars = 8;  // scalars[8], scalars[9]: dt', dbias of the last forward for upstream gradient 1
constexpr unsigned int kTraceLaunches = 4096;

int check_dbg(siglip_ctx* c, const char* where) {
  if (c->dbg_host != nullptr && c->dbg_host->code != 0) {
    char buf[320];
    const unsigned int code = c->dbg_host->code;
    const bool peer = (code >= 5);   // 5 text pull, 6 helper wait, 7 fold, 8 last-fold flag, 9 scalar exchange, 1x aux jobs
    snprintf(buf, sizeof(buf),
             "%s: device wait timed out at site %u (block %u thread %u aux %u %u %u)%s", where, code,
             c->dbg_host->block, c->dbg_host->thread, c->dbg_host->aux0, c->dbg_host->aux1, c->dbg_host->aux2,
             peer ? " — a peer rank did not reach the matching call within SIGLIP_OPT_PEER_TIMEOUT_MS" : "");
    return fail(SIGLIP_ERR_CUDA, buf);
  }
  return 0;
}

int timing_mark(siglip_ctx* c, std::vector<cudaEvent_t>& evs, size_t& used, cudaStream_t st) {
  if (!c->kernel_timing) return 0;
  if (used == evs.size()) {
    cudaEvent_t e;
    CK(cudaEventCreate(&e));
    evs.push_back(e);
  }
  CK(cudaEventRecord(evs[used++], st));
  return 0;
}

inline size_t chunk_stride(const siglip_ctx* c) { return static_cast<size_t>(c->Bmax) * c->D; }
inline unsigned long long peer_timeout_ns(const siglip_ctx* c) {
  return static_cast<unsigned long long>(c->peer_timeout_ms) * 1000000ull;
}

// Sigma operand + fp16 text copy number i, allocated on first use. The fused step needs two (own chunk, chunk in
// flight), the split forward / backward API one per text chunk (they all live from the forward to the backward).
int ensure_g(siglip_ctx* c, int i) {
  if (c->G[i] != nullptr) return 0;
  const size_t gbytes = static_cast<size_t>(c->Bp) * c->Bp * sizeof(__nv_bfloat16);
  const size_t tbytes = chunk_stride(c) * sizeof(__nv_bfloat16);
  cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&c->G[i]), gbytes);
  if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&c->txt16[i]), tbytes);
  if (e != cudaSuccess) {
    cudaGetLastError();
    if (c->G[i]) cudaFree(c->G[i]);
    c->G[i] = nullptr;
    char buf[256];
    snprintf(buf, sizeof(buf),
             "sigma operand %d needs %.2f GiB more device memory (B = %d: %d x %d 16-bit per text chunk kept for the "
             "backward; siglip_fwd_bwd needs 2 of them, the split forward/backward API one per rank): %s",
             i, static_cast<double>(gbytes + tbytes) / (1024.0 * 1024.0 * 1024.0), c->Bmax, c->Bp, c->Bp,
             cudaGetErrorString(e));
    return fail(SIGLIP_ERR_CUDA, buf);
  }
  c->workspace_bytes += gbytes + tbytes;
  return 0;
}

// Workspace of the gradient kernel's split-K (fp32 partial accumulators of the tiles of a ragged last wave): fewer than
// one 64 KiB partial per SM can ever be outstanding.
constexpr int kSplitKMaxTiles = 160;
int ensure_splitk(siglip_ctx* c) {
  if (c->splitk_ws != nullptr) return 0;
  const size_t bytes = static_cast<size_t>(c->num_sms + 2) * 128 * siglip::kTileCols * sizeof(float);
  CK(cudaMalloc(reinterpret_cast<void**>(&c->splitk_ws), bytes));
  CK(cudaMalloc(reinterpret_cast<void**>(&c->splitk_counters), 2 * kSplitKMaxTiles * sizeof(unsigned int)));
  CK(cudaMemset(c->splitk_counters, 0, 2 * kSplitKMaxTiles * sizeof(unsigned int)));
  c->splitk_ws_bytes = bytes;
  c->workspace_bytes += bytes;
  return 0;
}

struct AuxList {
  siglip::AuxJob jobs[siglip::kMaxAuxJobs];
  int n = 0;
  AuxList() { memset(jobs, 0, sizeof(jobs)); }
  siglip::AuxJob& add(int kind) {
    siglip::AuxJob& j = jobs[n++];
    j.kind = kind;
    return j;
  }
};

struct EndSignal {
  unsigned int* const* ptrs = nullptr;
  int n = 0;
  unsigned int value = 0;
};

void apply_aux(siglip_ctx* c, KernelParams& p, const AuxList& aux, const EndSignal& end) {
  p.naux = aux.n;
  for (int i = 0; i < aux.n; ++i) {
    p.aux[i] = aux.jobs[i];
    if (p.aux[i].sig_n > 0 || p.aux[i].done_flag != nullptr) p.aux[i].ticket = c->sync_words + i;
  }
  p.cvt_scale = kXScale;
  p.tprime_f64 = c->tprime_f64;
  p.pdl = c->pdl;
  p.peer_timeout_ns = peer_timeout_ns(c);
  if (end.n > 0 || c->aux_trace_on) {
    p.end_sig_ptrs = end.ptrs;
    p.end_sig_n = end.n;
    p.end_sig_value = end.value;
    p.end_ticket = c->sync_words + kSyncEndTicket;
  }
  if (c->aux_trace_on && c->aux_trace != nullptr && c->aux_trace_n < kTraceLaunches) {
    p.aux_trace = c->aux_trace + 16ull * c->aux_trace_n;
    c->aux_trace_n++;
  }
}

struct FinJob {   // last chunk of a forward: the loss kernel's last CTA writes the results
  float* loss = nullptr;
  float* dt_prime = nullptr;
  float* dbias = nullptr;
};

// The loss kernel over one text chunk (Bn rows, owner's batch): S = img @ txt_c^T on wgmma, fused
// scale/bias/log-sigmoid/reduce. save: also write the sigma operand G[gi] (+ g_diag on the own chunk); the fp16 copies
// the gradient kernel needs are auxiliary jobs built by the caller.
int run_loss_chunk(siglip_ctx* c, int gi, bool own, bool first, const void* img, const __nv_bfloat16* txt_c, int Bn,
                   const float* t_prime, const float* bias, bool save, const AuxList& aux, const FinJob* fin,
                   const EndSignal& end, cudaStream_t st) {
  const int cg = c->cta_group;
  int rc;
  if ((rc = ensure_g(c, save ? gi : 0))) return rc;
  __nv_bfloat16* G = c->G[save ? gi : 0];
  CUtensorMap tmA, tmB, tmG;
  if ((rc = encode_operand(&tmA, img, c->B, c->D, c->D, 0, 128))) return rc;
  const int mc = c->mcast;
  if ((rc = encode_operand(&tmB, txt_c, Bn, c->D, c->D, 0, siglip::b_box_rows_kmajor(siglip::cluster_size(cg, mc)))))
    return rc;
  // store map of the sigma operand: [B, Bn] inside the padded [Bp, Bp] buffer, one 16-row x 32-column slab per TMA store
  if ((rc = encode_bf16_2d(&tmG, G, (uint64_t)Bn, (uint64_t)c->B, (uint64_t)c->Bp, 32, 16,
                           CU_TENSOR_MAP_SWIZZLE_64B)))
    return rc;
  KernelParams p;
  memset(&p, 0, sizeof(p));
  p.nprob = 1;
  // fp32-input path: both operands are fp16(x * kXScale), the accumulator is kXScale^2 <img, txt>
  p.prob[0].ab_f16 = c->input_f16;
  p.s_scale = c->input_f16 ? 1.0f / (kXScale * kXScale) : 1.0f;
  p.prob[0].M = c->B;
  p.prob[0].N = Bn;
  p.prob[0].K = c->D;
  p.t_prime = t_prime;
  p.bias = bias;
  p.inv_b = 1.0f / static_cast<float>(c->B);
  p.G = G;
  p.ldg = c->Bp;
  p.g_diag = c->g_diag;
  p.own_chunk = own ? 1 : 0;
  p.store_g = save ? 1 : 0;
  p.g_scale = kGScale;
  p.partials = c->partials;
  p.accumulate_partials = first ? 0 : 1;  // the first chunk of a forward overwrites every slot of the grid
  if (fin != nullptr) {
    p.fin_counter = c->fin_counter;
    p.fin_loss = fin->loss;
    p.fin_dt_prime = fin->dt_prime;
    p.fin_dbias = fin->dbias;
  }
  p.dbg = c->dbg_dev;
  if (save && c->dbg_no_gstore) p.store_g = 0;  // timing experiments only (wrong gradients)
  apply_aux(c, p, aux, end);
  unsigned long long* wstats = nullptr;
  if (c->dbg_loss_waitstats) {   // diagnostic: where the roles of the loss kernel spend their cycles
    CK(cudaMalloc(reinterpret_cast<void**>(&wstats), 8 * 256 * sizeof(unsigned long long)));
    CK(cudaMemsetAsync(wstats, 0, 8 * 256 * sizeof(unsigned long long), st));
    p.wait_stats = wstats;
  }
  if ((rc = timing_mark(c, c->ev_loss, c->ev_loss_used, st))) return rc;
  CKI(siglip::launch_gemm(cg, siglip::kModeLoss, c->stages_loss, mc, &tmA, &tmB, &tmA, &tmB, &tmG, p, c->num_sms,
                          st));
  if ((rc = timing_mark(c, c->ev_loss, c->ev_loss_used, st))) return rc;
  if (wstats != nullptr) {
    CK(cudaStreamSynchronize(st));
    std::vector<unsigned long long> h(8 * 256);
    CK(cudaMemcpy(h.data(), wstats, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    // slots written by the kernel: [0] producer empty-wait, [1] consumer thread 0 full-wait, [3] its loop cycles
    double s[4] = {0, 0, 0, 0};
    int nall = 0;
    for (int b = 0; b < 256; ++b) {
      if (h[8 * b + 3]) nall++;
      for (int j = 0; j < 4; ++j) s[j] += static_cast<double>(h[8 * b + j]);
    }
    printf("[loss waitstats] %d CTAs: producer empty-wait %.0f cyc/CTA | consumer thread 0: loop %.0f cyc/CTA, "
           "waiting for operands %.1f%%\n",
           nall, s[0] / (nall ? nall : 1), s[3] / (nall ? nall : 1), 100.0 * s[1] / (s[3] > 0 ? s[3] : 1));
    fflush(stdout);
    cudaFree(wstats);
  }
  c->launches++;
  return 0;
}

// auxiliary jobs of a saving loss kernel: bf16 -> fp16 x 16 copies of the chunk's text (and, on the own chunk, of the
// images) for the gradient kernel
void add_cvt_jobs(siglip_ctx* c, AuxList& aux, int gi, bool own, const void* img, const __nv_bfloat16* txt_c, int Bn) {
  if (c->dbg_no_cvt) return;
  siglip::AuxJob& jt = aux.add(siglip::kAuxCvt);
  jt.src = reinterpret_cast<const uint4*>(txt_c);
  jt.dst = reinterpret_cast<uint4*>(c->txt16[gi]);
  jt.n16 = static_cast<unsigned long long>(Bn) * c->D * sizeof(__nv_bfloat16) / 16;
  jt.cvt_copy = c->input_f16;
  if (own) {
    siglip::AuxJob& ji = aux.add(siglip::kAuxCvt);
    ji.src = reinterpret_cast<const uint4*>(img);
    ji.dst = reinterpret_cast<uint4*>(c->img16);
    ji.n16 = static_cast<unsigned long long>(c->B) * c->D * sizeof(__nv_bfloat16) / 16;
    ji.cvt_copy = c->input_f16;
  }
}

struct GradOut {
  const float* dimg_add = nullptr;   // fp32 running dimg of the previous chunks (null: first chunk)
  void* dimg_out = nullptr;
  bool dimg_bf16 = false;
  const float* dtxt_add = nullptr;   // fp32 folded sum of the peers' contributions (last launch of the fused step)
  const unsigned int* dtxt_add_flag = nullptr;  // ... which must not be read before this local flag holds dtxt_add_value
  unsigned int dtxt_add_value = 0;
  void* dtxt_out = nullptr;
  bool dtxt_bf16 = false;
  float* sc_dt_prime = nullptr;      // backward of the two scalars rides on this launch
  float* sc_dbias = nullptr;
};

// The two gradient contractions of one chunk in one launch (g = upstream gradient, device scalar or null):
//   prob 0: dimg (+)= g (t/B) (G @ txt_c  [+ g_diag * txt_own])      A = G K-major,  B = txt16[gi] N-major     K = Bn
//   prob 1: dtxt_c  = g (t/B) (G^T @ img  [+ g_diag * img])          A = G M-major,  B = img16 N-major         K = B
int run_grad_chunk(siglip_ctx* c, int gi, bool own, const void* img, const __nv_bfloat16* txt_own, int Bn,
                   const float* t_prime, const float* grad_out, const GradOut& o, const AuxList& aux,
                   const EndSignal& end, cudaStream_t st) {
  const int cg = c->cta_group;
  const int bk = siglip::b_box_k_mnmajor(siglip::cluster_size(cg, c->mcast));
  CUtensorMap tmA0, tmB0, tmA1, tmB1;
  int rc;
  if (c->G[gi] == nullptr) return fail(SIGLIP_ERR_STATE, "gradient kernel without a saved sigma operand");
  if ((rc = encode_operand(&tmA0, c->G[gi], c->B, Bn, c->Bp, 0, 128))) return rc;
  if ((rc = encode_operand(&tmB0, c->txt16[gi], c->D, Bn, c->D, 1, 0, bk))) return rc;
  if ((rc = encode_operand(&tmA1, c->G[gi], Bn, c->B, c->Bp, 1, 0))) return rc;
  if ((rc = encode_operand(&tmB1, c->img16, c->D, c->B, c->D, 1, 0, bk))) return rc;
  KernelParams p;
  memset(&p, 0, sizeof(p));
  p.nprob = 2;
  for (int i = 0; i < 2; ++i) {
    Problem& pr = p.prob[i];
    pr.N = c->D;
    pr.b_mn = 1;
    pr.ab_f16 = 1;
    pr.acc_scale = 1.0f / (kGScale * kXScale);
    pr.ldo = c->D;
    pr.ldx = c->D;
    pr.fix_vec = own ? c->g_diag : nullptr;
    pr.fix_f16 = c->saved_f16;
    pr.fix_mat_scale = c->saved_f16 ? 1.0f / kXScale : 1.0f;
  }
  p.prob[0].M = c->B;
  p.prob[0].K = Bn;
  p.prob[0].a_mn = 0;
  p.prob[0].out = o.dimg_out;
  p.prob[0].out_bf16 = o.dimg_bf16 ? 1 : 0;
  p.prob[0].add_src = o.dimg_add;
  p.prob[0].ld_add = c->D;
  p.prob[0].fix_mat = own ? txt_own : nullptr;
  p.prob[1].M = Bn;
  p.prob[1].K = c->B;
  p.prob[1].a_mn = 1;
  p.prob[1].out = o.dtxt_out;
  p.prob[1].out_bf16 = o.dtxt_bf16 ? 1 : 0;
  p.prob[1].add_src = o.dtxt_add;
  p.prob[1].ld_add = c->D;
  p.prob[1].fix_mat = own ? reinterpret_cast<const __nv_bfloat16*>(img) : nullptr;
  p.p1_wait_flag = o.dtxt_add_flag;
  p.p1_wait_value = o.dtxt_add_value;
  if (o.sc_dt_prime != nullptr || o.sc_dbias != nullptr) {
    p.sc_saved = c->scalars + kSavedScalars;
    p.sc_dt_prime = o.sc_dt_prime;
    p.sc_dbias = o.sc_dbias;
  }
  p.t_prime = t_prime;
  p.grad_out = grad_out;
  p.inv_b = 1.0f / static_cast<float>(c->B);
  p.dbg = c->dbg_dev;
  if (c->split_k != 0 && c->mcast == 1) {
    if ((rc = ensure_splitk(c))) return rc;
    p.sk_request = c->split_k;
    p.sk_ws = c->splitk_ws;
    p.sk_ws_bytes = c->splitk_ws_bytes;
    p.sk_counters = c->splitk_counters;
    p.sk_max_tiles = kSplitKMaxTiles;
  }
  apply_aux(c, p, aux, end);
  if ((rc = timing_mark(c, c->ev_grad, c->ev_grad_used, st))) return rc;
  CKI(siglip::launch_gemm(cg, siglip::kModeOut, c->stages_grad, c->mcast, &tmA0, &tmB0, &tmA1, &tmB1,
                          &tmA0, p, c->num_sms, st));
  if ((rc = timing_mark(c, c->ev_grad, c->ev_grad_used, st))) return rc;
  c->launches++;
  return 0;
}

// Owner of the text chunk a rank scores at step k. Unidirectional: r, r+1, r+2, ... (the pairs of the reference's ring,
// rwightman_sigmoid_loss.py:108-122). Bidirectional: r, r+1, r-1, r+2, r-2, ... (the order of its bidir exchange,
// rwightman_sigmoid_loss.py:75-107). At every step each owner is read by exactly one rank either way.
inline int step_offset(const siglip_ctx* c, int k) {
  if (!c->bidir) return k;
  return (k & 1) ? (k + 1) / 2 : -(k / 2);
}
inline int step_owner(const siglip_ctx* c, int rank, int k) {
  return ((rank + step_offset(c, k)) % c->world + c->world) % c->world;
}

int signal_peers(siglip_ctx* c, int kind, unsigned int value, cudaStream_t st) {
  CKI(siglip::launch_signal_flags(c->signal_ptrs_dev + kind * c->world, c->world, value, st));
  c->launches++;
  return 0;
}

int wait_peers(siglip_ctx* c, int kind, unsigned int value, cudaStream_t st) {
  CKI(siglip::launch_wait_flags(c->flags + kind * kMaxWorld, c->world, value, peer_timeout_ns(c), c->dbg_dev, st));
  c->launches++;
  return 0;
}

int wait_one(siglip_ctx* c, int kind, int rank, unsigned int value, cudaStream_t st) {
  CKI(siglip::launch_wait_flags(c->flags + kind * kMaxWorld + rank, 1, value, peer_timeout_ns(c), c->dbg_dev, st));
  c->launches++;
  return 0;
}

inline EndSignal end_signal(siglip_ctx* c, int kind, unsigned int value) {
  EndSignal e;
  e.ptrs = c->signal_ptrs_dev + kind * c->world;
  e.n = c->world;
  e.value = value;
  return e;
}

int check_call(siglip_ctx* c, const void* img, const void* txt, const float* t_prime, cudaStream_t st) {
  if (c == nullptr || img == nullptr || txt == nullptr || t_prime == nullptr)
    return fail(SIGLIP_ERR_INVALID, "null argument");
  if (c->world > 1 && !c->peers_ready)
    return fail(SIGLIP_ERR_STATE, "world > 1 but peer handles were not imported (siglip_ctx_import_handles)");
  if (c->world > 1) {
    // a multi-rank step cannot be replayed from a CUDA graph: the flag values its kernels wait for / raise are kernel
    // parameters that advance with every step (a single-rank step has none and captures fine)
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cs) == cudaSuccess && cs != cudaStreamCaptureStatusNone)
      return fail(SIGLIP_ERR_STATE,
                  "a multi-rank step cannot be captured into a CUDA graph (its cross-rank flag values advance every step)");
  }
  return 0;
}

// pull of the text chunk of step k (owner o) into my gathered buffer, as an auxiliary job of the kernel of step k-1
void add_pull_job(siglip_ctx* c, AuxList& aux, int o, unsigned int s) {
  siglip::AuxJob& j = aux.add(siglip::kAuxCopy);
  j.src = reinterpret_cast<const uint4*>(c->peer_txt[o] + o * chunk_stride(c));
  j.dst = reinterpret_cast<uint4*>(c->txt_all + o * chunk_stride(c));
  j.n16 = static_cast<unsigned long long>(c->Bs[o]) * c->D * sizeof(__nv_bfloat16) / 16;
  j.wait_flags = c->flags + 0 * kMaxWorld + o;
  j.wait_n = 1;
  j.wait_value = s;
  j.site = 5;
}

// ---------------------------------------------------------------------------------------------------------------
// Forward (split API): W loss kernels. Step k scores my images against the text chunk owned by rank (r + k) % W — the
// pairs the reference's ring covers (rwightman_sigmoid_loss.py:108-122) without the hop-by-hop forwarding: every chunk
// is pulled straight from its owner through the NVSwitch by the idle warps of the loss kernel of the previous step.
// With save the W sigma operands stay in the context until the backward (O(W B^2) memory: the fused step needs O(B^2)).
// ---------------------------------------------------------------------------------------------------------------
int forward_impl(siglip_ctx* c, const void* img, const void* txt, const float* t_prime, const float* bias, float* loss,
                 bool save, cudaStream_t st) {
  int rc;
  if ((rc = check_call(c, img, txt, t_prime, st))) return rc;
  if (bias == nullptr || loss == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if ((rc = check_dbg(c, "siglip forward (previous launch)"))) return rc;
  CK(cudaSetDevice(c->device));
  const int W = c->world, r = c->rank;
  const size_t stride = chunk_stride(c);
  const unsigned int s = ++c->n_fwd;
  // the saved state is being overwritten (a forward without save still replaces my gathered text slot, which the
  // backward of a multi-rank job reads for the positive-pair term); valid again once a saving forward is enqueued
  if (save || c->world > 1) c->gen = 0;

  const __nv_bfloat16* own_txt = reinterpret_cast<const __nv_bfloat16*>(txt);
  if (W > 1) {
    // peers must have finished pulling my text slot in their previous forward before I overwrite it
    if ((rc = wait_peers(c, 2, s - 1, st))) return rc;
    CK(cudaMemcpyAsync(c->txt_all + r * stride, txt, static_cast<size_t>(c->B) * c->D * sizeof(__nv_bfloat16),
                       cudaMemcpyDeviceToDevice, st));
    if ((rc = signal_peers(c, 0, s, st))) return rc;
    own_txt = c->txt_all + r * stride;
  }
  // loss, and (for backward) dt' / dbias for an upstream gradient of 1: written by the last CTA of the last chunk
  FinJob fin;
  fin.loss = loss;
  fin.dt_prime = save ? c->scalars + kSavedScalars : nullptr;
  fin.dbias = save ? c->scalars + kSavedScalars + 1 : nullptr;
  for (int k = 0; k < W; ++k) {
    const int cidx = step_owner(c, r, k);
    const __nv_bfloat16* txt_c = (k == 0) ? own_txt : c->txt_all + cidx * stride;
    if (save && (rc = ensure_g(c, k))) return rc;
    AuxList aux;
    if (save) add_cvt_jobs(c, aux, k, k == 0, img, txt_c, c->Bs[cidx]);
    if (k + 1 < W) {
      const int nxt = step_owner(c, r, k + 1);
      if (c->overlap_pull) {
        add_pull_job(c, aux, nxt, s);
      } else {
        // un-overlapped variant (A/B measurements): wait + copy as separate stream operations
        if ((rc = wait_one(c, 0, nxt, s, st))) return rc;
        CK(cudaMemcpyAsync(c->txt_all + nxt * stride, c->peer_txt[nxt] + nxt * stride,
                           static_cast<size_t>(c->Bs[nxt]) * c->D * sizeof(__nv_bfloat16), cudaMemcpyDefault, st));
      }
    }
    if ((rc = run_loss_chunk(c, k, k == 0, k == 0, img, txt_c, c->Bs[cidx], t_prime, bias, save, aux,
                             (k == W - 1) ? &fin : nullptr, EndSignal(), st)))
      return rc;
  }
  if (W > 1) {
    if ((rc = signal_peers(c, 2, s, st))) return rc;
  }
  CK(cudaGetLastError());
  if (save) {
    c->saved_f16 = c->input_f16;
    static unsigned long long next_gen = 0;
    c->gen = ++next_gen;
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Backward (split API): W gradient kernels over the sigma operands the forward saved, the OWN chunk last. Gradient slot
// j = 1..W handles step k = j (j < W) or k = 0 (j == W). My contribution to owner (r + k) % W goes to a local fp32 slot
// and is published with flag value (n-1) W + j; one slot later the owner folds it into its accumulator from inside its
// own gradient kernel (P2P loads over NVSwitch), so every remote contribution has a whole gradient kernel of slack and
// only a local add remains at the end: this is all_gather's backward (reduce-scatter SUM, torch functional.py:343-354;
// reverse ring, distributed_utils.py:75-77, 94-98) without an exposed collective.
// ---------------------------------------------------------------------------------------------------------------
int backward_impl(siglip_ctx* c, const void* img, const void* txt, const float* t_prime, const float* grad_out,
                  void* dimg, void* dtxt, float* dt_prime, float* dbias, cudaStream_t st) {
  int rc;
  if ((rc = check_call(c, img, txt, t_prime, st))) return rc;
  if (dimg == nullptr || dtxt == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (c->gen == 0) return fail(SIGLIP_ERR_STATE, "no forward state saved for backward (call siglip_forward with save = 1)");
  if ((rc = check_dbg(c, "siglip backward (previous launch)"))) return rc;
  CK(cudaSetDevice(c->device));
  const int W = c->world, r = c->rank;
  const size_t stride = chunk_stride(c);
  const unsigned int n = ++c->n_bwd;
  const unsigned int base = (n - 1) * static_cast<unsigned int>(W);
  if (W > 1 && c->prewait3 + 1 < n + 0u) {
    // peers must have finished reading my contribution slots of the previous backward before I overwrite them
    if ((rc = wait_peers(c, 3, n - 1, st))) return rc;
    c->prewait3 = n - 1;
  }
  // bf16 text of the own chunk (positive-pair term of dimg): my gathered slot, or the caller's tensor for one rank
  const __nv_bfloat16* own_txt =
      (W > 1) ? c->txt_all + r * stride : reinterpret_cast<const __nv_bfloat16*>(txt);
  for (int j = 1; j <= W; ++j) {
    const int k = (j < W) ? j : 0;
    const int cidx = step_owner(c, r, k);
    const bool last = (j == W);
    GradOut o;
    o.dimg_add = (j > 1) ? c->dimg_acc : nullptr;
    o.dimg_out = last ? dimg : static_cast<void*>(c->dimg_acc);
    o.dimg_bf16 = last && c->grad_bf16;
    o.dtxt_out = (W == 1) ? dtxt : static_cast<void*>(c->slots + cidx * stride);
    o.dtxt_bf16 = (W == 1) && c->grad_bf16;
    AuxList aux;
    if (W > 1 && c->overlap_reduce && j >= 2) {
      // the contribution for me that rank p = r - offset(j-1) produced in ITS gradient slot j-1
      const int pr = ((r - step_offset(c, j - 1)) % W + W) % W;
      siglip::AuxJob& f = aux.add(siglip::kAuxFold);
      f.src = reinterpret_cast<const uint4*>(c->peer_slots[pr] + r * stride);
      f.src2 = (j == 2) ? nullptr : reinterpret_cast<const uint4*>(c->dtxt_acc);
      f.dst = reinterpret_cast<uint4*>(c->dtxt_acc);
      f.n16 = static_cast<unsigned long long>(c->B) * c->D * sizeof(float) / 16;
      f.wait_flags = c->flags + 1 * kMaxWorld + pr;
      f.wait_n = 1;
      f.wait_value = base + static_cast<unsigned int>(j - 1);
      f.site = 7;
    }
    // dt' / dbias = saved * grad_out is written by the last gradient launch (the in-kernel mean over ranks, when
    // enabled, is a separate one-warp kernel below)
    const bool scalars_here = last && !(W > 1 && c->sync_scalar_grads);
    o.sc_dt_prime = scalars_here ? dt_prime : nullptr;
    o.sc_dbias = scalars_here ? dbias : nullptr;
    if ((rc = run_grad_chunk(c, k, k == 0, img, own_txt, c->Bs[cidx], t_prime, grad_out, o, aux, EndSignal(), st)))
      return rc;
    if (W > 1 && (!last || !c->overlap_reduce)) {
      if ((rc = signal_peers(c, 1, base + static_cast<unsigned int>(j), st))) return rc;
    }
  }
  if (W > 1) {
    if (c->overlap_reduce) {
      // dtxt = (sum of the W-1 remote contributions, already local) + my own contribution: a local add
      CKI(siglip::launch_reduce_slots(dtxt, c->grad_bf16, c->final_ptrs_dev, 2, static_cast<size_t>(c->B) * c->D,
                                      c->num_sms, st));
    } else {
      if ((rc = wait_peers(c, 1, base + static_cast<unsigned int>(W), st))) return rc;
      CKI(siglip::launch_reduce_slots(dtxt, c->grad_bf16, c->reduce_ptrs_dev, W, static_cast<size_t>(c->B) * c->D,
                                      c->num_sms, st));
    }
    c->launches++;
    if ((rc = signal_peers(c, 3, n, st))) return rc;
  }
  if (W > 1 && c->sync_scalar_grads) {
    // a collective: issued on every rank whether or not this caller wants the two values. My mailbox is free again:
    // every peer has signalled the text of a later forward, i.e. finished the backward that read it.
    CKI(siglip::launch_allreduce_scalars(c->scalars + kSavedScalars, grad_out,
                                         reinterpret_cast<float*>(c->flags + kMailboxOffset), c->mailbox_ptrs_dev,
                                         c->signal_ptrs_dev + 4 * W, c->flags + 4 * kMaxWorld, W, n, dt_prime, dbias,
                                         c->tprime_f64, peer_timeout_ns(c), c->dbg_dev, st));
    c->launches++;
  }
  CK(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// The fused step (siglip_fwd_bwd): loss AND all four gradients of one training step, chunk by chunk, with TWO sigma
// operands however many ranks there are. Launch order for W chunks (L = loss kernel, G = gradient kernel; index = step
// k of the chunk schedule, 0 = own chunk):
//        L0  L1 G1  L2 G2  ...  L(W-1) G(W-1)  G0
// L0 keeps its sigma operand (buffer 0) to the very end — the own chunk must be the LAST gradient slot so that every
// remote dtxt contribution has a whole gradient kernel of slack before its owner folds it — every other chunk's
// operand lives in buffer 1 from its loss kernel to the gradient kernel right behind it. The exchange of the split API
// (text pulls inside L(k-1), progressive fold inside G(j+1)) is unchanged, but every flag is waited for / raised INSIDE
// these kernels (auxiliary warps, last-CTA tickets): a multi-rank step is exactly 2W launches, like a single-rank one.
// The last gradient launch adds the folded peer contributions in its dtxt epilogue, so there is no reduction kernel.
// ---------------------------------------------------------------------------------------------------------------
int fused_impl(siglip_ctx* c, const void* img, const void* txt, const float* t_prime, const float* bias, float* loss,
               const float* grad_out, void* dimg, void* dtxt, float* dt_prime, float* dbias, cudaStream_t st) {
  int rc;
  if ((rc = check_call(c, img, txt, t_prime, st))) return rc;
  if (bias == nullptr || loss == nullptr || dimg == nullptr || dtxt == nullptr)
    return fail(SIGLIP_ERR_INVALID, "null argument");
  if ((rc = check_dbg(c, "siglip_fwd_bwd (previous launch)"))) return rc;
  CK(cudaSetDevice(c->device));
  const int W = c->world, r = c->rank;
  const size_t stride = chunk_stride(c);
  const unsigned int s = ++c->n_fwd;
  const unsigned int n = ++c->n_bwd;
  const unsigned int base = (n - 1) * static_cast<unsigned int>(W);
  const bool ik = c->inkernel_sync != 0;
  c->gen = 0;                       // the sigma operands of a split forward (if any) are overwritten
  c->saved_f16 = c->input_f16;
  if ((rc = ensure_g(c, 0))) return rc;
  if (W > 1 && (rc = ensure_g(c, 1))) return rc;
  const __nv_bfloat16* own_txt = reinterpret_cast<const __nv_bfloat16*>(txt);
  const size_t own_bytes = static_cast<size_t>(c->B) * c->D * sizeof(__nv_bfloat16);
  FinJob fin;
  fin.loss = loss;
  fin.dt_prime = c->scalars + kSavedScalars;
  fin.dbias = c->scalars + kSavedScalars + 1;

  // ---- L0: own chunk. Its auxiliary warps also publish my text to the peers and start the first pull ----
  {
    AuxList aux;
    if (W > 1) {
      if (ik) {
        // my gathered slot is what the peers pull: they must be done with the previous forward's copy (flag 2),
        // then "text of forward s in place" (flag 0) goes to every rank once all CTAs have copied their share
        siglip::AuxJob& cp = aux.add(siglip::kAuxCopy);
        cp.src = reinterpret_cast<const uint4*>(txt);
        cp.dst = reinterpret_cast<uint4*>(c->txt_all + r * stride);
        cp.n16 = own_bytes / 16;
        cp.wait_flags = c->flags + 2 * kMaxWorld;
        cp.wait_n = W;
        cp.wait_value = s - 1;
        cp.site = 11;
        cp.sig_ptrs = c->signal_ptrs_dev + 0 * W;
        cp.sig_n = W;
        cp.sig_value = s;
      } else {
        if ((rc = wait_peers(c, 2, s - 1, st))) return rc;
        CK(cudaMemcpyAsync(c->txt_all + r * stride, txt, own_bytes, cudaMemcpyDeviceToDevice, st));
        if ((rc = signal_peers(c, 0, s, st))) return rc;
      }
    }
    add_cvt_jobs(c, aux, 0, true, img, own_txt, c->B);
    if (W > 1) {
      if (ik) {
        // my contribution slots of the previous backward must have been read by their owners (flag 3) before G1
        // overwrites the first of them
        siglip::AuxJob& w3 = aux.add(siglip::kAuxWaitOnly);
        w3.wait_flags = c->flags + 3 * kMaxWorld;
        w3.wait_n = W;
        w3.wait_value = n - 1;
        w3.site = 13;
      } else if (c->prewait3 + 1 < n) {
        if ((rc = wait_peers(c, 3, n - 1, st))) return rc;
      }
      c->prewait3 = n - 1;
      add_pull_job(c, aux, step_owner(c, r, 1), s);
    }
    if ((rc = run_loss_chunk(c, 0, true, true, img, own_txt, c->B, t_prime, bias, true, aux, (W == 1) ? &fin : nullptr,
                             EndSignal(), st)))
      return rc;
  }
  if (W > 1) own_txt = c->txt_all + r * stride;   // the copy the peers see (same bytes)
  // ---- remote chunks: L_k then G_k (gradient slot j = k) ----
  for (int k = 1; k < W; ++k) {
    const int cidx = step_owner(c, r, k);
    const __nv_bfloat16* txt_c = c->txt_all + cidx * stride;
    {
      AuxList aux;
      add_cvt_jobs(c, aux, 1, false, img, txt_c, c->Bs[cidx]);
      if (k + 1 < W) add_pull_job(c, aux, step_owner(c, r, k + 1), s);
      const bool lastL = (k == W - 1);
      EndSignal end = (lastL && ik) ? end_signal(c, 2, s) : EndSignal();   // "I have pulled everyone's text"
      if ((rc = run_loss_chunk(c, 1, false, false, img, txt_c, c->Bs[cidx], t_prime, bias, true, aux,
                               lastL ? &fin : nullptr, end, st)))
        return rc;
      if (lastL && !ik && (rc = signal_peers(c, 2, s, st))) return rc;
    }
    const int j = k;
    GradOut o;
    o.dimg_add = (j > 1) ? c->dimg_acc : nullptr;
    o.dimg_out = c->dimg_acc;
    o.dtxt_out = c->slots + cidx * stride;
    AuxList aux;
    if (j >= 2) {
      const int pr = ((r - step_offset(c, j - 1)) % W + W) % W;
      siglip::AuxJob& f = aux.add(siglip::kAuxFold);
      f.src = reinterpret_cast<const uint4*>(c->peer_slots[pr] + r * stride);
      f.src2 = (j == 2) ? nullptr : reinterpret_cast<const uint4*>(c->dtxt_acc);
      f.dst = reinterpret_cast<uint4*>(c->dtxt_acc);
      f.n16 = static_cast<unsigned long long>(c->B) * c->D * sizeof(float) / 16;
      f.wait_flags = c->flags + 1 * kMaxWorld + pr;
      f.wait_n = 1;
      f.wait_value = base + static_cast<unsigned int>(j - 1);
      f.site = 7;
    }
    EndSignal end = ik ? end_signal(c, 1, base + static_cast<unsigned int>(j)) : EndSignal();
    if ((rc = run_grad_chunk(c, 1, false, img, own_txt, c->Bs[cidx], t_prime, grad_out, o, aux, end, st))) return rc;
    if (!ik && (rc = signal_peers(c, 1, base + static_cast<unsigned int>(j), st))) return rc;
  }
  // ---- G0: own chunk, gradient slot W. Folds the last remote contribution and adds the folded sum in its epilogue ----
  {
    GradOut o;
    o.dimg_add = (W > 1) ? c->dimg_acc : nullptr;
    o.dimg_out = dimg;
    o.dimg_bf16 = c->grad_bf16 != 0;
    o.dtxt_out = dtxt;
    o.dtxt_bf16 = c->grad_bf16 != 0;
    AuxList aux;
    if (W > 1) {
      const int pr = ((r - step_offset(c, W - 1)) % W + W) % W;
      siglip::AuxJob& f = aux.add(siglip::kAuxFold);
      f.src = reinterpret_cast<const uint4*>(c->peer_slots[pr] + r * stride);
      f.src2 = (W == 2) ? nullptr : reinterpret_cast<const uint4*>(c->dtxt_acc);
      f.dst = reinterpret_cast<uint4*>(c->dtxt_acc);
      f.n16 = static_cast<unsigned long long>(c->B) * c->D * sizeof(float) / 16;
      f.wait_flags = c->flags + 1 * kMaxWorld + pr;
      f.wait_n = 1;
      f.wait_value = base + static_cast<unsigned int>(W - 1);
      f.site = 7;
      f.done_flag = c->sync_words + kSyncFoldDone;
      f.done_value = n;
      o.dtxt_add = c->dtxt_acc;
      o.dtxt_add_flag = c->sync_words + kSyncFoldDone;
      o.dtxt_add_value = n;
    }
    const bool scalars_here = !(W > 1 && c->sync_scalar_grads);
    o.sc_dt_prime = scalars_here ? dt_prime : nullptr;
    o.sc_dbias = scalars_here ? dbias : nullptr;
    EndSignal end = (W > 1 && ik) ? end_signal(c, 3, n) : EndSignal();   // "I have read everyone's contributions"
    if ((rc = run_grad_chunk(c, 0, true, img, own_txt, c->B, t_prime, grad_out, o, aux, end, st))) return rc;
    if (W > 1 && !ik && (rc = signal_peers(c, 3, n, st))) return rc;
  }
  if (W > 1 && c->sync_scalar_grads) {
    CKI(siglip::launch_allreduce_scalars(c->scalars + kSavedScalars, grad_out,
                                         reinterpret_cast<float*>(c->flags + kMailboxOffset), c->mailbox_ptrs_dev,
                                         c->signal_ptrs_dev + 4 * W, c->flags + 4 * kMaxWorld, W, n, dt_prime, dbias,
                                         c->tprime_f64, peer_timeout_ns(c), c->dbg_dev, st));
    c->launches++;
  }
  CK(cudaGetLastError());
  return 0;
}

void free_ctx(siglip_ctx* c);

}  // namespace

extern "C" {

const char* siglip_version(void) { return "siglip_b200 0.5.0 sm_90a"; }

const char* siglip_last_error(void) { return g_last_error.c_str(); }

int siglip_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  int ok = 0;
  for (int i = 0; i < n; ++i) {
    int major = 0;
    if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, i) == cudaSuccess && major == 9) ok++;
  }
  return ok;
}

static int ctx_create_impl(siglip_ctx** out, int device, int rank, int world, const int* Bs, int D) {
  if (out == nullptr) return fail(SIGLIP_ERR_INVALID, "out is null");
  *out = nullptr;
  if (world < 1 || world > kMaxWorld || rank < 0 || rank >= world)
    return fail(SIGLIP_ERR_INVALID, "rank/world out of range (world <= 32)");
  int Bmax = 0;
  for (int p = 0; p < world; ++p) {
    if (Bs[p] < 1) return fail(SIGLIP_ERR_INVALID, "need B >= 1 on every rank");
    Bmax = Bs[p] > Bmax ? Bs[p] : Bmax;
  }
  if (D < 8 || (D % 8) != 0) return fail(SIGLIP_ERR_INVALID, "need D a positive multiple of 8");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return fail(SIGLIP_ERR_NO_DEVICE, "no CUDA device visible; this library has no CPU fallback");
  }
  if (device < 0 || device >= ndev) return fail(SIGLIP_ERR_INVALID, "device ordinal out of range");
  int major = 0;
  CK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
  if (major != 9) return fail(SIGLIP_ERR_NO_DEVICE, "device is not compute capability 9.x (H100, sm_90a required)");
  CK(cudaSetDevice(device));
  siglip_ctx* c = new siglip_ctx();
  // every failure below releases what was allocated so far (the caller never sees a half-built context)
  struct Guard {
    siglip_ctx* c;
    ~Guard() {
      if (c != nullptr) free_ctx(c);
    }
  } guard{c};
  c->device = device;
  c->rank = rank;
  c->world = world;
  for (int p = 0; p < world; ++p) c->Bs[p] = Bs[p];
  c->B = Bs[rank];
  c->Bmax = Bmax;
  c->D = D;
  c->Bp = round_up(Bmax, 256);
  c->dbg_no_gstore = getenv("SIGLIP_DEBUG_NO_GSTORE") != nullptr;
  c->dbg_no_cvt = getenv("SIGLIP_DEBUG_NO_CVT") != nullptr;
  c->dbg_loss_waitstats = getenv("SIGLIP_DEBUG_LOSS_WAITSTATS") != nullptr;
  if (const char* e = getenv("SIGLIP_INKERNEL_SYNC")) c->inkernel_sync = atoi(e) ? 1 : 0;   // A/B measurements
  if (const char* e = getenv("SIGLIP_SPLIT_K")) c->split_k = atoi(e);
  if (const char* e = getenv("SIGLIP_PDL")) c->pdl = atoi(e) ? 1 : 0;
  if (const char* e = getenv("SIGLIP_PEER_TIMEOUT_MS")) {
    const long long v = atoll(e);
    if (v > 0) c->peer_timeout_ms = v;
  }
  CK(cudaDeviceGetAttribute(&c->num_sms, cudaDevAttrMultiProcessorCount, device));
  const size_t stride = chunk_stride(c);
  size_t total = 0;
  auto alloc = [&](void** p, size_t bytes) -> cudaError_t {
    cudaError_t e = cudaMalloc(p, bytes);
    if (e == cudaSuccess) {
      total += bytes;
      e = cudaMemset(*p, 0, bytes);
    }
    return e;
  };
  CK(alloc(reinterpret_cast<void**>(&c->g_diag), static_cast<size_t>(c->Bp) * sizeof(float)));
  CK(alloc(reinterpret_cast<void**>(&c->img16), static_cast<size_t>(c->B) * D * sizeof(__nv_bfloat16)));
  CK(alloc(reinterpret_cast<void**>(&c->partials), static_cast<size_t>(c->num_sms) * 4 * sizeof(double)));
  CK(alloc(reinterpret_cast<void**>(&c->fin_counter), sizeof(unsigned int)));
  CK(alloc(reinterpret_cast<void**>(&c->flags), kFlagBytes));
  CK(alloc(reinterpret_cast<void**>(&c->sync_words), kSyncWords * sizeof(unsigned int)));
  CK(alloc(reinterpret_cast<void**>(&c->scalars), 24 * sizeof(float)));
  if (world > 1) {
    CK(alloc(reinterpret_cast<void**>(&c->txt_all), stride * world * sizeof(__nv_bfloat16)));
    CK(alloc(reinterpret_cast<void**>(&c->slots), stride * world * sizeof(float)));
    CK(alloc(reinterpret_cast<void**>(&c->dimg_acc), static_cast<size_t>(c->B) * D * sizeof(float)));
    CK(alloc(reinterpret_cast<void**>(&c->dtxt_acc), static_cast<size_t>(c->B) * D * sizeof(float)));
    CK(alloc(reinterpret_cast<void**>(&c->reduce_ptrs_dev), world * sizeof(float*)));
    CK(alloc(reinterpret_cast<void**>(&c->final_ptrs_dev), 2 * sizeof(float*)));
    CK(alloc(reinterpret_cast<void**>(&c->signal_ptrs_dev), kFlagKinds * world * sizeof(unsigned int*)));
    CK(alloc(reinterpret_cast<void**>(&c->mailbox_ptrs_dev), world * sizeof(float*)));
    const float* fin[2] = {c->dtxt_acc, c->slots + rank * stride};
    CK(cudaMemcpy(c->final_ptrs_dev, fin, sizeof(fin), cudaMemcpyHostToDevice));
  }
  CK(cudaHostAlloc(reinterpret_cast<void**>(&c->dbg_host), sizeof(DebugRecord), cudaHostAllocMapped));
  memset(c->dbg_host, 0, sizeof(DebugRecord));
  CK(cudaHostGetDevicePointer(reinterpret_cast<void**>(&c->dbg_dev), c->dbg_host, 0));
  c->peer_txt[rank] = c->txt_all;
  c->peer_slots[rank] = c->slots;
  c->peer_flags[rank] = c->flags;
  c->workspace_bytes = total;
  int rc = ensure_g(c, 0);
  if (rc) return rc;
  CK(cudaDeviceSynchronize());
  guard.c = nullptr;
  *out = c;
  return 0;
}

int siglip_ctx_create(siglip_ctx** out, int device, int rank, int world, int B, int D) {
  if (world < 1 || world > kMaxWorld) return fail(SIGLIP_ERR_INVALID, "rank/world out of range (world <= 32)");
  int Bs[kMaxWorld];
  for (int p = 0; p < world; ++p) Bs[p] = B;
  return ctx_create_impl(out, device, rank, world, Bs, D);
}

int siglip_ctx_create_uneven(siglip_ctx** out, int device, int rank, int world, const int* batch_per_rank, int D) {
  if (batch_per_rank == nullptr) return fail(SIGLIP_ERR_INVALID, "batch_per_rank is null");
  if (world < 1 || world > kMaxWorld) return fail(SIGLIP_ERR_INVALID, "rank/world out of range (world <= 32)");
  return ctx_create_impl(out, device, rank, world, batch_per_rank, D);
}

int siglip_ctx_set_option(siglip_ctx* c, int option, int value) {
  if (c == nullptr) return fail(SIGLIP_ERR_INVALID, "ctx is null");
  switch (option) {
    case SIGLIP_OPT_CTA_GROUP:
      if (value != 1 && value != 2) return fail(SIGLIP_ERR_INVALID, "cta_group must be 1 or 2");
      c->cta_group = value;
      return 0;
    case SIGLIP_OPT_OVERLAP_PULL:
      c->overlap_pull = value ? 1 : 0;
      return 0;
    case SIGLIP_OPT_OVERLAP_REDUCE:
      c->overlap_reduce = value ? 1 : 0;
      return 0;
    case SIGLIP_OPT_GRAD_BF16:
      c->grad_bf16 = value ? 1 : 0;
      return 0;
    case SIGLIP_OPT_MCAST:
      if (value != 1 && value != 2) return fail(SIGLIP_ERR_INVALID, "mcast must be 1 or 2");
      c->mcast = value;
      return 0;
    case SIGLIP_OPT_EPI_SLEEP_GRAD_NS:   // accepted for existing callers; no effect on sm_90a (see the header)
    case SIGLIP_OPT_EPI_SLEEP_LOSS_NS:
      return 0;
    case SIGLIP_OPT_GRAD_TILE_N:         // accepted for existing callers; every column tile is 128 wide on sm_90a
      if (value != 0 && value != 128 && value != 256) return fail(SIGLIP_ERR_INVALID, "grad_tile_n must be 0, 128 or 256");
      return 0;
    case SIGLIP_OPT_INPUT_F16:
      c->input_f16 = value ? 1 : 0;
      return 0;
    case SIGLIP_OPT_BIDIR:
      c->bidir = value ? 1 : 0;
      c->gen = 0;   // a saved forward was laid out in the other order
      return 0;
    case SIGLIP_OPT_SYNC_SCALAR_GRADS:
      c->sync_scalar_grads = value ? 1 : 0;
      return 0;
    case SIGLIP_OPT_STAGES_LOSS:
    case SIGLIP_OPT_STAGES_GRAD:
      if (value != 0 && value != 4 && value != 6) return fail(SIGLIP_ERR_INVALID, "pipeline stages must be 0 (default), 4 or 6");
      (option == SIGLIP_OPT_STAGES_LOSS ? c->stages_loss : c->stages_grad) = value;
      return 0;
    case SIGLIP_OPT_KERNEL_TIMING:
      c->kernel_timing = value ? 1 : 0;
      c->ev_loss_used = c->ev_grad_used = 0;
      return 0;
    case SIGLIP_OPT_PEER_TIMEOUT_MS:
      if (value < 1) return fail(SIGLIP_ERR_INVALID, "peer timeout must be >= 1 ms");
      c->peer_timeout_ms = value;
      return 0;
    case SIGLIP_OPT_INKERNEL_SYNC:
      c->inkernel_sync = value ? 1 : 0;
      return 0;
    case SIGLIP_OPT_SPLIT_K:
      if (value < -1 || value == 1 || value > 8) return fail(SIGLIP_ERR_INVALID, "split_k must be -1 (auto), 0 (off) or 2..8");
      c->split_k = value;
      return 0;
    case SIGLIP_OPT_TPRIME_F64:
      c->tprime_f64 = value ? 1 : 0;
      return 0;
    case SIGLIP_OPT_PDL:
      c->pdl = value ? 1 : 0;
      return 0;
    case SIGLIP_OPT_AUX_TRACE:
      c->aux_trace_on = value ? 1 : 0;
      c->aux_trace_n = 0;
      if (value && c->aux_trace == nullptr) {
        CK(cudaSetDevice(c->device));
        CK(cudaMalloc(reinterpret_cast<void**>(&c->aux_trace), kTraceLaunches * 16 * sizeof(unsigned long long)));
      }
      if (value) {
        std::vector<unsigned long long> init(static_cast<size_t>(kTraceLaunches) * 16, 0ull);
        for (unsigned int i = 0; i < kTraceLaunches; ++i)
          init[16ull * i + 8] = init[16ull * i + 10] = init[16ull * i + 13] = ~0ull;  // minima
        CK(cudaMemcpy(c->aux_trace, init.data(), init.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice));
      }
      return 0;
    default:
      return fail(SIGLIP_ERR_INVALID, "unknown option");
  }
}

size_t siglip_ctx_workspace_bytes(const siglip_ctx* c) { return c ? c->workspace_bytes : 0; }

size_t siglip_ctx_handle_bytes(void) { return sizeof(IpcBlob); }

int siglip_ctx_export_handles(siglip_ctx* c, void* out_bytes, size_t capacity) {
  if (c == nullptr || out_bytes == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (capacity < sizeof(IpcBlob)) return fail(SIGLIP_ERR_INVALID, "handle buffer too small");
  if (c->world == 1) return fail(SIGLIP_ERR_STATE, "world == 1 has no peers to export to");
  CK(cudaSetDevice(c->device));
  IpcBlob b;
  memset(&b, 0, sizeof(b));
  CK(cudaIpcGetMemHandle(&b.txt, c->txt_all));
  CK(cudaIpcGetMemHandle(&b.slots, c->slots));
  CK(cudaIpcGetMemHandle(&b.flags, c->flags));
  b.rank = c->rank;
  b.device = c->device;
  b.B = c->B;
  b.D = c->D;
  b.Bmax = c->Bmax;
  if (gethostname(b.host, sizeof(b.host) - 1) != 0) b.host[0] = 0;
  memcpy(out_bytes, &b, sizeof(b));
  return 0;
}

static int publish_peer_tables(siglip_ctx* c) {
  const size_t stride = chunk_stride(c);
  std::vector<const float*> red(c->world);
  for (int p = 0; p < c->world; ++p) red[p] = c->peer_slots[p] + c->rank * stride;
  CK(cudaMemcpy(c->reduce_ptrs_dev, red.data(), c->world * sizeof(float*), cudaMemcpyHostToDevice));
  std::vector<unsigned int*> sig(kFlagKinds * c->world);
  for (int k = 0; k < kFlagKinds; ++k)
    for (int p = 0; p < c->world; ++p)
      sig[k * c->world + p] = c->peer_flags[p] + k * kMaxWorld + (c->loopback ? p : c->rank);
  CK(cudaMemcpy(c->signal_ptrs_dev, sig.data(), sig.size() * sizeof(unsigned int*), cudaMemcpyHostToDevice));
  std::vector<const float*> mb(c->world);
  for (int p = 0; p < c->world; ++p) {
    mb[p] = reinterpret_cast<const float*>(c->peer_flags[p] + kMailboxOffset);
    // loopback: the "peers'" mailboxes are separate words a test can seed (siglip_debug_set_mailbox)
    if (c->loopback && p != c->rank) mb[p] = c->loop_mailboxes + 2 * p;
  }
  CK(cudaMemcpy(c->mailbox_ptrs_dev, mb.data(), c->world * sizeof(float*), cudaMemcpyHostToDevice));
  c->peers_ready = true;
  return 0;
}

int siglip_ctx_import_handles(siglip_ctx* c, const void* all_ranks_bytes, size_t bytes_per_rank) {
  if (c == nullptr || all_ranks_bytes == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (bytes_per_rank != sizeof(IpcBlob)) return fail(SIGLIP_ERR_INVALID, "bytes_per_rank != siglip_ctx_handle_bytes()");
  if (c->world == 1) return fail(SIGLIP_ERR_STATE, "world == 1 has no peers to import");
  CK(cudaSetDevice(c->device));
  const char* base = static_cast<const char*>(all_ranks_bytes);
  for (int p = 0; p < c->world; ++p) {
    IpcBlob b;
    memcpy(&b, base + static_cast<size_t>(p) * bytes_per_rank, sizeof(b));
    if (b.rank != p) return fail(SIGLIP_ERR_INVALID, "handle blobs are not ordered by rank");
    if (b.B != c->Bs[p] || b.D != c->D || b.Bmax != c->Bmax)
      return fail(SIGLIP_ERR_INVALID,
                  "peer context has a different batch / D than this rank was told: every rank must be created with the "
                  "same D and the same per-rank batch list (equal batches unless siglip_ctx_create_uneven)");
    if (p == c->rank) continue;
    char me[64] = {0};
    if (gethostname(me, sizeof(me) - 1) != 0) me[0] = 0;
    if (strncmp(me, b.host, sizeof(me)) != 0) {
      char buf[384];
      snprintf(buf, sizeof(buf),
               "rank %d runs on host '%s', this rank (%d) on '%s': the text / gradient exchange goes through CUDA-IPC "
               "peer mappings over NVLink and is limited to the ranks of ONE node (one NVSwitch domain, world <= %d). "
               "For a multi-node job give the loss a per-node process group (group=) and reduce across nodes outside.",
               p, b.host, c->rank, me, kMaxWorld);
      return fail(SIGLIP_ERR_INVALID, buf);
    }
    void *pt = nullptr, *ps = nullptr, *pf = nullptr;
    cudaError_t oe = cudaIpcOpenMemHandle(&pt, b.txt, cudaIpcMemLazyEnablePeerAccess);
    if (oe == cudaSuccess) oe = cudaIpcOpenMemHandle(&ps, b.slots, cudaIpcMemLazyEnablePeerAccess);
    if (oe == cudaSuccess) oe = cudaIpcOpenMemHandle(&pf, b.flags, cudaIpcMemLazyEnablePeerAccess);
    if (oe != cudaSuccess) {
      cudaGetLastError();
      char buf[384];
      snprintf(buf, sizeof(buf),
               "cannot map the buffers of rank %d (its CUDA device %d) into rank %d: %s. The ranks of one context must be "
               "GPUs of the same node with peer (NVLink / PCIe P2P) access to each other, one process per GPU.",
               p, b.device, c->rank, cudaGetErrorString(oe));
      return fail(SIGLIP_ERR_CUDA, buf);
    }
    c->peer_txt[p] = static_cast<__nv_bfloat16*>(pt);
    c->peer_slots[p] = static_cast<float*>(ps);
    c->peer_flags[p] = static_cast<unsigned int*>(pf);
  }
  return publish_peer_tables(c);
}

int siglip_forward(siglip_ctx* c, const void* img, const void* txt, const float* t_prime, const float* bias,
                   float* loss, int save_for_backward, void* cuda_stream) {
  return forward_impl(c, img, txt, t_prime, bias, loss, save_for_backward != 0, static_cast<cudaStream_t>(cuda_stream));
}

unsigned long long siglip_ctx_saved_generation(const siglip_ctx* c) { return c ? c->gen : 0ull; }

int siglip_backward(siglip_ctx* c, const void* img, const void* txt, const float* t_prime, const float* grad_out,
                    void* dimg, void* dtxt, float* dt_prime, float* dbias, void* cuda_stream) {
  return backward_impl(c, img, txt, t_prime, grad_out, dimg, dtxt, dt_prime, dbias,
                       static_cast<cudaStream_t>(cuda_stream));
}

int siglip_fwd_bwd(siglip_ctx* c, const void* img, const void* txt, const float* t_prime, const float* bias,
                   float* loss, void* dimg, void* dtxt, float* dt_prime, float* dbias, void* cuda_stream) {
  if (dimg == nullptr || dtxt == nullptr || dt_prime == nullptr || dbias == nullptr)
    return fail(SIGLIP_ERR_INVALID, "null gradient pointer");
  return fused_impl(c, img, txt, t_prime, bias, loss, nullptr, dimg, dtxt, dt_prime, dbias,
                    static_cast<cudaStream_t>(cuda_stream));
}

int siglip_fwd_bwd_scaled(siglip_ctx* c, const void* img, const void* txt, const float* t_prime, const float* bias,
                          const float* grad_out, float* loss, void* dimg, void* dtxt, float* dt_prime, float* dbias,
                          void* cuda_stream) {
  if (dimg == nullptr || dtxt == nullptr || dt_prime == nullptr || dbias == nullptr)
    return fail(SIGLIP_ERR_INVALID, "null gradient pointer");
  return fused_impl(c, img, txt, t_prime, bias, loss, grad_out, dimg, dtxt, dt_prime, dbias,
                    static_cast<cudaStream_t>(cuda_stream));
}

int siglip_fwd(siglip_ctx* c, const void* img, const void* txt, const float* t_prime, const float* bias, float* loss,
               void* cuda_stream) {
  return siglip_forward(c, img, txt, t_prime, bias, loss, 0, cuda_stream);
}

// device scalars of host-entry set s: t', bias, loss, dt', dbias
static inline float* host_set_scalars(siglip_ctx* c, int s) { return c->scalars + (s ? 10 : 0); }

static int host_entry_init(siglip_ctx* c, bool with_grads) {
  const size_t chunk_elems = static_cast<size_t>(c->B) * c->D;
  if (c->h_img[0] == nullptr) {
    for (int s = 0; s < 2; ++s) {
      CK(cudaMalloc(reinterpret_cast<void**>(&c->h_img[s]), chunk_elems * sizeof(__nv_bfloat16)));
      CK(cudaMalloc(reinterpret_cast<void**>(&c->h_txt[s]), chunk_elems * sizeof(__nv_bfloat16)));
      CK(cudaEventCreateWithFlags(&c->ev_h2d[s], cudaEventDisableTiming));
      CK(cudaEventCreateWithFlags(&c->ev_step[s], cudaEventDisableTiming));
      CK(cudaEventCreateWithFlags(&c->ev_done[s], cudaEventDisableTiming));
    }
    CK(cudaMalloc(reinterpret_cast<void**>(&c->h_dimg), chunk_elems * sizeof(float)));
    CK(cudaMalloc(reinterpret_cast<void**>(&c->h_dtxt), chunk_elems * sizeof(float)));
    CK(cudaHostAlloc(reinterpret_cast<void**>(&c->h_pinned), 16 * sizeof(float), cudaHostAllocDefault));
    CK(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&c->d2h_stream, cudaStreamNonBlocking));
    c->workspace_bytes += chunk_elems * (4 * sizeof(__nv_bfloat16) + 2 * sizeof(float));
  }
  if (with_grads && c->h_gimg[0] == nullptr) {
    for (int s = 0; s < 2; ++s) {
      CK(cudaMalloc(reinterpret_cast<void**>(&c->h_gimg[s]), chunk_elems * sizeof(__nv_bfloat16)));
      CK(cudaMalloc(reinterpret_cast<void**>(&c->h_gtxt[s]), chunk_elems * sizeof(__nv_bfloat16)));
    }
    c->workspace_bytes += chunk_elems * 4 * sizeof(__nv_bfloat16);
  }
  return 0;
}

// Enqueue one end-to-end step: the host->device copies of ITS inputs go to an internal copy stream into staging set
// (ticket & 1), the step runs on the caller's stream once they have landed, its results are copied to (pinned) host
// memory behind it on a second copy stream: (loss, dt', dbias) always, the bf16 gradients when host buffers are given.
// With two staging sets the copies of step n+1 (and the gradient read-back of step n) overlap the kernels.
int siglip_host_submit_grads(siglip_ctx* c, const void* img_host, const void* txt_host, float t_prime, float bias,
                             void* dimg_host_bf16, void* dtxt_host_bf16, unsigned long long* ticket,
                             void* cuda_stream) {
  if (c == nullptr || img_host == nullptr || txt_host == nullptr || ticket == nullptr)
    return fail(SIGLIP_ERR_INVALID, "null argument");
  if ((dimg_host_bf16 == nullptr) != (dtxt_host_bf16 == nullptr))
    return fail(SIGLIP_ERR_INVALID, "give both gradient host buffers or neither");
  const bool with_grads = dimg_host_bf16 != nullptr;
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  CK(cudaSetDevice(c->device));
  int rc;
  if ((rc = host_entry_init(c, with_grads))) return rc;
  const size_t chunk_bytes = static_cast<size_t>(c->B) * c->D * sizeof(__nv_bfloat16);
  const unsigned long long n = c->host_submitted;
  const int s = static_cast<int>(n & 1);
  if (n >= 2) {
    // set s was used by step n-2: its kernels and read-back must be done before the staging buffers are overwritten,
    // and the caller must have collected its results (siglip_host_wait) before the pinned slot is reused
    CK(cudaStreamWaitEvent(c->copy_stream, c->ev_done[s], 0));
    CK(cudaEventSynchronize(c->ev_done[s]));
  }
  float* pin = c->h_pinned + 8 * s;
  pin[0] = t_prime;
  pin[1] = bias;
  float* sc = host_set_scalars(c, s);
  CK(cudaMemcpyAsync(sc, pin, 2 * sizeof(float), cudaMemcpyHostToDevice, c->copy_stream));
  CK(cudaMemcpyAsync(c->h_img[s], img_host, chunk_bytes, cudaMemcpyHostToDevice, c->copy_stream));
  CK(cudaMemcpyAsync(c->h_txt[s], txt_host, chunk_bytes, cudaMemcpyHostToDevice, c->copy_stream));
  CK(cudaEventRecord(c->ev_h2d[s], c->copy_stream));
  CK(cudaStreamWaitEvent(st, c->ev_h2d[s], 0));
  const int saved_bf16 = c->grad_bf16, saved_fmt = c->input_f16, saved_tp64 = c->tprime_f64;
  c->grad_bf16 = with_grads ? 1 : 0;  // gradients that travel back are bf16 (what autograd returns for bf16 inputs)
  c->input_f16 = 0;                   // ... from bf16 host buffers
  c->tprime_f64 = 0;                  // the staged scalars are fp32
  void* gi = with_grads ? static_cast<void*>(c->h_gimg[s]) : static_cast<void*>(c->h_dimg);
  void* gt = with_grads ? static_cast<void*>(c->h_gtxt[s]) : static_cast<void*>(c->h_dtxt);
  rc = siglip_fwd_bwd(c, c->h_img[s], c->h_txt[s], sc + 0, sc + 1, sc + 2, gi, gt, sc + 3, sc + 4, st);
  c->grad_bf16 = saved_bf16;
  c->input_f16 = saved_fmt;
  c->tprime_f64 = saved_tp64;
  if (rc) return rc;
  CK(cudaEventRecord(c->ev_step[s], st));
  CK(cudaStreamWaitEvent(c->d2h_stream, c->ev_step[s], 0));
  CK(cudaMemcpyAsync(pin + 4, sc + 2, 3 * sizeof(float), cudaMemcpyDeviceToHost, c->d2h_stream));
  if (with_grads) {
    CK(cudaMemcpyAsync(dimg_host_bf16, c->h_gimg[s], chunk_bytes, cudaMemcpyDeviceToHost, c->d2h_stream));
    CK(cudaMemcpyAsync(dtxt_host_bf16, c->h_gtxt[s], chunk_bytes, cudaMemcpyDeviceToHost, c->d2h_stream));
  }
  CK(cudaEventRecord(c->ev_done[s], c->d2h_stream));
  c->host_submitted = n + 1;
  *ticket = n;
  return 0;
}

int siglip_host_submit(siglip_ctx* c, const void* img_host, const void* txt_host, float t_prime, float bias,
                       unsigned long long* ticket, void* cuda_stream) {
  return siglip_host_submit_grads(c, img_host, txt_host, t_prime, bias, nullptr, nullptr, ticket, cuda_stream);
}

int siglip_host_wait(siglip_ctx* c, unsigned long long ticket, float* loss_host, float* dt_prime_host,
                     float* dbias_host) {
  if (c == nullptr || loss_host == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (ticket >= c->host_submitted || ticket + 2 < c->host_submitted)
    return fail(SIGLIP_ERR_STATE, "ticket is not one of the last two submitted steps");
  CK(cudaSetDevice(c->device));
  const int s = static_cast<int>(ticket & 1);
  CK(cudaEventSynchronize(c->ev_done[s]));
  int rc;
  if ((rc = check_dbg(c, "siglip_host_wait"))) return rc;
  const float* pin = c->h_pinned + 8 * s;
  *loss_host = pin[4];
  if (dt_prime_host) *dt_prime_host = pin[5];
  if (dbias_host) *dbias_host = pin[6];
  return 0;
}

int siglip_fwd_bwd_host(siglip_ctx* c, const void* img_host, const void* txt_host, float t_prime, float bias,
                        float* loss_host, float* dimg_host, float* dtxt_host, float* dt_prime_host,
                        float* dbias_host, void* cuda_stream) {
  if (loss_host == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  unsigned long long ticket = 0;
  int rc = siglip_host_submit(c, img_host, txt_host, t_prime, bias, &ticket, cuda_stream);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  const size_t chunk_elems = static_cast<size_t>(c->B) * c->D;
  if (dimg_host) CK(cudaMemcpyAsync(dimg_host, c->h_dimg, chunk_elems * sizeof(float), cudaMemcpyDeviceToHost, st));
  if (dtxt_host) CK(cudaMemcpyAsync(dtxt_host, c->h_dtxt, chunk_elems * sizeof(float), cudaMemcpyDeviceToHost, st));
  if ((rc = siglip_host_wait(c, ticket, loss_host, dt_prime_host, dbias_host))) return rc;
  if (dimg_host || dtxt_host) CK(cudaStreamSynchronize(st));
  return 0;
}

int siglip_ctx_kernel_times(siglip_ctx* c, double* loss_ms, int* loss_launches, double* grad_ms, int* grad_launches) {
  if (c == nullptr) return fail(SIGLIP_ERR_INVALID, "ctx is null");
  CK(cudaSetDevice(c->device));
  CK(cudaDeviceSynchronize());
  double tl = 0.0, tg = 0.0;
  for (size_t i = 0; i + 1 < c->ev_loss_used; i += 2) {
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, c->ev_loss[i], c->ev_loss[i + 1]));
    tl += ms;
  }
  for (size_t i = 0; i + 1 < c->ev_grad_used; i += 2) {
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, c->ev_grad[i], c->ev_grad[i + 1]));
    tg += ms;
  }
  if (getenv("SIGLIP_DEBUG_PRINT_TIMES")) {  // per-launch durations of the last W loss / gradient launches
    std::string s = "[kernel times rank " + std::to_string(c->rank) + "] loss:";
    char b[32];
    const size_t nl = c->ev_loss_used / 2, ng = c->ev_grad_used / 2;
    for (size_t i = (nl > (size_t)c->world ? nl - c->world : 0); i < nl; ++i) {
      float ms = 0.f;
      cudaEventElapsedTime(&ms, c->ev_loss[2 * i], c->ev_loss[2 * i + 1]);
      snprintf(b, sizeof(b), " %.3f", ms);
      s += b;
    }
    s += " | grad:";
    for (size_t i = (ng > (size_t)c->world ? ng - c->world : 0); i < ng; ++i) {
      float ms = 0.f;
      cudaEventElapsedTime(&ms, c->ev_grad[2 * i], c->ev_grad[2 * i + 1]);
      snprintf(b, sizeof(b), " %.3f", ms);
      s += b;
    }
    printf("%s\n", s.c_str());
    fflush(stdout);
  }
  if (loss_ms) *loss_ms = tl;
  if (grad_ms) *grad_ms = tg;
  if (loss_launches) *loss_launches = static_cast<int>(c->ev_loss_used / 2);
  if (grad_launches) *grad_launches = static_cast<int>(c->ev_grad_used / 2);
  c->ev_loss_used = c->ev_grad_used = 0;
  return 0;
}

int siglip_debug_loopback(siglip_ctx* c) {
  if (c == nullptr) return fail(SIGLIP_ERR_INVALID, "ctx is null");
  if (c->world == 1) return fail(SIGLIP_ERR_STATE, "loopback needs world > 1");
  CK(cudaSetDevice(c->device));
  // the "peers'" contributions to my text gradient: a zero buffer, so that the step's dtxt output is exactly this
  // rank's own-chunk contribution; the "peers'" scalar mailboxes: separate words a test can seed
  const size_t stride = chunk_stride(c);
  if (c->loop_zero == nullptr) {
    CK(cudaMalloc(reinterpret_cast<void**>(&c->loop_zero), stride * c->world * sizeof(float)));
    CK(cudaMemset(c->loop_zero, 0, stride * c->world * sizeof(float)));
    CK(cudaMalloc(reinterpret_cast<void**>(&c->loop_mailboxes), 2 * kMaxWorld * sizeof(float)));
    CK(cudaMemset(c->loop_mailboxes, 0, 2 * kMaxWorld * sizeof(float)));
  }
  for (int p = 0; p < c->world; ++p) {
    c->peer_txt[p] = c->txt_all;
    c->peer_slots[p] = (p == c->rank) ? c->slots : c->loop_zero;
    c->peer_flags[p] = c->flags;
  }
  c->loopback = true;   // every signal then raises the flag entry of EVERY rank in the local table
  return publish_peer_tables(c);
}

int siglip_debug_set_text_chunk(siglip_ctx* c, int chunk, const void* txt_dev, void* cuda_stream) {
  if (c == nullptr || txt_dev == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (c->world == 1 || chunk < 0 || chunk >= c->world) return fail(SIGLIP_ERR_INVALID, "chunk out of range");
  CK(cudaMemcpyAsync(c->txt_all + chunk * chunk_stride(c), txt_dev,
                     static_cast<size_t>(c->Bs[chunk]) * c->D * sizeof(__nv_bfloat16), cudaMemcpyDeviceToDevice,
                     static_cast<cudaStream_t>(cuda_stream)));
  return 0;
}

int siglip_debug_get_slot(siglip_ctx* c, int chunk, float* out_dev, void* cuda_stream) {
  if (c == nullptr || out_dev == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (c->world == 1 || chunk < 0 || chunk >= c->world) return fail(SIGLIP_ERR_INVALID, "chunk out of range");
  CK(cudaMemcpyAsync(out_dev, c->slots + chunk * chunk_stride(c),
                     static_cast<size_t>(c->Bs[chunk]) * c->D * sizeof(float), cudaMemcpyDeviceToDevice,
                     static_cast<cudaStream_t>(cuda_stream)));
  return 0;
}

int siglip_debug_set_mailbox(siglip_ctx* c, int peer, float dt_prime, float dbias) {
  if (c == nullptr) return fail(SIGLIP_ERR_INVALID, "ctx is null");
  if (!c->loopback || peer < 0 || peer >= c->world || peer == c->rank)
    return fail(SIGLIP_ERR_INVALID, "siglip_debug_set_mailbox needs a loopback context and a peer rank != own rank");
  CK(cudaSetDevice(c->device));
  const float v[2] = {dt_prime, dbias};
  CK(cudaMemcpy(c->loop_mailboxes + 2 * peer, v, sizeof(v), cudaMemcpyHostToDevice));
  return 0;
}

int siglip_ctx_aux_trace(siglip_ctx* c, unsigned long long* out, int max_launches, int* n_launches) {
  if (c == nullptr || out == nullptr || n_launches == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  CK(cudaSetDevice(c->device));
  CK(cudaDeviceSynchronize());
  int n = static_cast<int>(c->aux_trace_n);
  if (n > max_launches) n = max_launches;
  if (n > 0) CK(cudaMemcpy(out, c->aux_trace, static_cast<size_t>(n) * 16 * sizeof(unsigned long long),
                           cudaMemcpyDeviceToHost));
  *n_launches = n;
  c->aux_trace_n = 0;
  return 0;
}

int siglip_normalize_fwd(siglip_ctx* c, const void* x, int in_bf16, void* xhat_bf16, float* inv_norm,
                         void* cuda_stream) {
  if (c == nullptr || x == nullptr || xhat_bf16 == nullptr || inv_norm == nullptr)
    return fail(SIGLIP_ERR_INVALID, "null argument");
  if ((reinterpret_cast<uintptr_t>(x) & 15u) || (reinterpret_cast<uintptr_t>(xhat_bf16) & 15u))
    return fail(SIGLIP_ERR_INVALID, "buffers must be 16-byte aligned");
  CK(cudaSetDevice(c->device));
  CKI(siglip::launch_normalize_fwd(x, in_bf16, static_cast<__nv_bfloat16*>(xhat_bf16), inv_norm, c->B, c->D,
                                   c->input_f16 ? kXScale : 0.0f, c->num_sms, static_cast<cudaStream_t>(cuda_stream)));
  c->launches++;
  return 0;
}

int siglip_convert_f32(siglip_ctx* c, const float* x_f32, void* out_16bit, void* cuda_stream) {
  if (c == nullptr || x_f32 == nullptr || out_16bit == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if ((reinterpret_cast<uintptr_t>(x_f32) & 15u) || (reinterpret_cast<uintptr_t>(out_16bit) & 15u))
    return fail(SIGLIP_ERR_INVALID, "buffers must be 16-byte aligned");
  CK(cudaSetDevice(c->device));
  CKI(siglip::launch_convert_f32(x_f32, out_16bit, static_cast<size_t>(c->B) * c->D, c->input_f16 ? kXScale : 0.0f,
                                 c->num_sms, static_cast<cudaStream_t>(cuda_stream)));
  c->launches++;
  return 0;
}

int siglip_normalize_bwd(siglip_ctx* c, const void* x, int in_bf16, const float* inv_norm, const void* dxhat,
                         int grad_bf16, void* dx, void* cuda_stream) {
  if (c == nullptr || x == nullptr || inv_norm == nullptr || dxhat == nullptr || dx == nullptr)
    return fail(SIGLIP_ERR_INVALID, "null argument");
  if ((reinterpret_cast<uintptr_t>(x) & 15u) || (reinterpret_cast<uintptr_t>(dxhat) & 15u) ||
      (reinterpret_cast<uintptr_t>(dx) & 15u))
    return fail(SIGLIP_ERR_INVALID, "buffers must be 16-byte aligned");
  CK(cudaSetDevice(c->device));
  CKI(siglip::launch_normalize_bwd(x, in_bf16, inv_norm, dxhat, grad_bf16, dx, c->B, c->D, c->num_sms,
                                   static_cast<cudaStream_t>(cuda_stream)));
  c->launches++;
  return 0;
}

int siglip_scale(siglip_ctx* c, const void* src, void* dst, size_t nbytes, int is_bf16, const float* g,
                 void* cuda_stream) {
  if (c == nullptr || src == nullptr || dst == nullptr || g == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  const size_t esz = is_bf16 ? 2 : 4;
  if ((nbytes % esz) != 0) return fail(SIGLIP_ERR_INVALID, "siglip_scale: nbytes is not a whole number of elements");
  CK(cudaSetDevice(c->device));
  CKI(siglip::launch_scale(src, dst, is_bf16, g, nbytes, c->num_sms, static_cast<cudaStream_t>(cuda_stream)));
  c->launches++;
  return 0;
}

unsigned long long siglip_ctx_launch_count(const siglip_ctx* c) { return c ? c->launches : 0ull; }

int siglip_debug_gemm(int device, int cta_group, int M, int N, int K, const void* A, long long lda, int a_mn,
                      const void* Bm, long long ldb, int b_mn, float* C, long long ldc, void* cuda_stream) {
  return siglip_debug_gemm_timed(device, cta_group, M, N, K, A, lda, a_mn, Bm, ldb, b_mn, C, ldc, 1, nullptr,
                                 cuda_stream);
}

int siglip_debug_gemm_timed(int device, int cta_group, int M, int N, int K, const void* A, long long lda, int a_mn,
                            const void* Bm, long long ldb, int b_mn, float* C, long long ldc, int iters,
                            float* ms_per_iter, void* cuda_stream) {
  if (A == nullptr || Bm == nullptr || C == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (cta_group != 1 && cta_group != 2) return fail(SIGLIP_ERR_INVALID, "cta_group must be 1 or 2");
  if (M < 1 || N < 8 || K < 1 || (N % 8) != 0) return fail(SIGLIP_ERR_INVALID, "need N % 8 == 0");
  if (siglip_device_count() == 0) return fail(SIGLIP_ERR_NO_DEVICE, "no sm_90 device; no CPU fallback");
  CK(cudaSetDevice(device));
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  int num_sms = 0;
  CK(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, device));
  CUtensorMap tmA, tmB;
  int rc;
  const bool fp8 = getenv("SIGLIP_DEBUG_AB_FP8") != nullptr;   // A, B hold e4m3 bytes, K-major
  const char* env_mc = getenv("SIGLIP_DEBUG_MCAST");
  const int mcast = env_mc ? atoi(env_mc) : 1;
  if (mcast != 1 && mcast != 2) return fail(SIGLIP_ERR_INVALID, "SIGLIP_DEBUG_MCAST must be 1 or 2");
  if (fp8) {
    if (a_mn || b_mn || mcast != 1) return fail(SIGLIP_ERR_INVALID, "the fp8 measurement path is K-major, no multicast");
    if ((rc = encode_u8_kmajor(&tmA, A, M, K, lda, 128))) return rc;
    if ((rc = encode_u8_kmajor(&tmB, Bm, N, K, ldb, siglip::b_box_rows_kmajor(cta_group)))) return rc;
  } else {
    const int cs = siglip::cluster_size(cta_group, mcast);
    if ((rc = encode_operand(&tmA, A, M, K, lda, a_mn, 128))) return rc;
    if ((rc = encode_operand(&tmB, Bm, N, K, ldb, b_mn, siglip::b_box_rows_kmajor(cs), siglip::b_box_k_mnmajor(cs))))
      return rc;
  }
  float* zero = nullptr;  // t' = 0 -> scale exp(0) * 1 = 1
  CK(cudaMalloc(reinterpret_cast<void**>(&zero), sizeof(float)));
  CK(cudaMemsetAsync(zero, 0, sizeof(float), st));
  DebugRecord* dbg_host = nullptr;
  DebugRecord* dbg_dev = nullptr;
  CK(cudaHostAlloc(reinterpret_cast<void**>(&dbg_host), sizeof(DebugRecord), cudaHostAllocMapped));
  memset(dbg_host, 0, sizeof(DebugRecord));
  CK(cudaHostGetDevicePointer(reinterpret_cast<void**>(&dbg_dev), dbg_host, 0));
  KernelParams p;
  memset(&p, 0, sizeof(p));
  p.nprob = 1;
  p.prob[0].M = M;
  p.prob[0].N = N;
  p.prob[0].K = K;
  p.prob[0].a_mn = a_mn ? 1 : 0;
  p.prob[0].b_mn = b_mn ? 1 : 0;
  p.prob[0].ab_f16 = fp8 ? 2 : (getenv("SIGLIP_DEBUG_AB_F16") ? 1 : 0);
  p.prob[0].acc_scale = 1.0f;
  p.prob[0].out = C;
  p.prob[0].ldo = ldc;
  p.t_prime = zero;
  p.inv_b = 1.0f;
  p.dbg = dbg_dev;
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  int lrc = 0;
  unsigned long long* wstats = nullptr;
  if (getenv("SIGLIP_DEBUG_WAITSTATS")) {
    printf("[waitstats cg=%d] max co-resident clusters: %d (SMs %d)\n", cta_group,
           siglip::query_max_active_clusters(siglip::cluster_size(cta_group, mcast)), num_sms);
    CK(cudaMalloc(reinterpret_cast<void**>(&wstats), 8 * 256 * sizeof(unsigned long long)));
    CK(cudaMemsetAsync(wstats, 0, 8 * 256 * sizeof(unsigned long long), st));
    p.wait_stats = wstats;
  }
  const char* env_st = getenv("SIGLIP_DEBUG_STAGES");
  const int stages = env_st ? atoi(env_st) : 0;
  if (stages != 0 && stages != 4 && stages != 6) return fail(SIGLIP_ERR_INVALID, "SIGLIP_DEBUG_STAGES must be 4 or 6");
  if (iters > 1)  // warm-up
    lrc = siglip::launch_gemm(cta_group, siglip::kModeOut, stages, mcast, &tmA, &tmB, &tmA, &tmB, &tmA, p, num_sms, st);
  cudaEventRecord(e0, st);
  for (int it = 0; it < iters && lrc == 0; ++it)
    lrc = siglip::launch_gemm(cta_group, siglip::kModeOut, stages, mcast, &tmA, &tmB, &tmA, &tmB, &tmA, p, num_sms, st);
  cudaEventRecord(e1, st);
  cudaError_t se = cudaStreamSynchronize(st);
  if (ms_per_iter != nullptr && se == cudaSuccess && lrc == 0) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    *ms_per_iter = ms / static_cast<float>(iters > 0 ? iters : 1);
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  if (wstats != nullptr) {
    std::vector<unsigned long long> h(8 * 256);
    cudaMemcpy(h.data(), wstats, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
    // slots written by the kernel: [0] producer empty-wait, [1] consumer thread 0 full-wait, [3] its loop cycles
    double s[4] = {0, 0, 0, 0};
    int nall = 0;
    for (int b = 0; b < 256; ++b) {
      if (h[8 * b + 3]) nall++;
      for (int j = 0; j < 4; ++j) s[j] += static_cast<double>(h[8 * b + j]);
    }
    printf("[waitstats cg=%d] %d CTAs: producer empty-wait %.0f cyc/CTA | consumer thread 0: loop %.0f cyc/CTA, "
           "waiting for operands %.1f%%\n",
           cta_group, nall, s[0] / (nall ? nall : 1), s[3] / (nall ? nall : 1), 100.0 * s[1] / (s[3] > 0 ? s[3] : 1));
    fflush(stdout);
    cudaFree(wstats);
  }
  int result = 0;
  if (dbg_host->code != 0) {
    char buf[256];
    snprintf(buf, sizeof(buf), "debug gemm: device wait timed out at site %u (block %u thread %u aux %u %u %u)",
             dbg_host->code, dbg_host->block, dbg_host->thread, dbg_host->aux0, dbg_host->aux1, dbg_host->aux2);
    result = fail(SIGLIP_ERR_CUDA, buf);
  } else if (lrc != 0) {
    result = fail(SIGLIP_ERR_CUDA, std::string("debug gemm launch failed: ") +
                                       cudaGetErrorString(static_cast<cudaError_t>(lrc)));
  } else if (se != cudaSuccess) {
    result = fail(SIGLIP_ERR_CUDA, std::string("debug gemm execution failed: ") + cudaGetErrorString(se));
  }
  cudaFreeHost(dbg_host);
  cudaFree(zero);
  return result;
}

void siglip_ctx_destroy(siglip_ctx* c) {
  if (c == nullptr) return;
  free_ctx(c);
}

}  // extern "C"

namespace {

void free_ctx(siglip_ctx* c) {
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  if (!c->loopback) {
    for (int p = 0; p < c->world; ++p) {
      if (p == c->rank) continue;
      if (c->peer_txt[p]) cudaIpcCloseMemHandle(c->peer_txt[p]);
      if (c->peer_slots[p]) cudaIpcCloseMemHandle(c->peer_slots[p]);
      if (c->peer_flags[p]) cudaIpcCloseMemHandle(c->peer_flags[p]);
    }
  }
  cudaFree(c->txt_all);
  for (int k = 0; k < kMaxWorld; ++k) {
    cudaFree(c->G[k]);
    cudaFree(c->txt16[k]);
  }
  cudaFree(c->g_diag);
  cudaFree(c->img16);
  cudaFree(c->slots);
  cudaFree(c->dimg_acc);
  cudaFree(c->dtxt_acc);
  cudaFree(c->final_ptrs_dev);
  cudaFree(c->partials);
  cudaFree(c->fin_counter);
  cudaFree(c->flags);
  cudaFree(c->sync_words);
  cudaFree(c->loop_mailboxes);
  cudaFree(c->loop_zero);
  cudaFree(c->scalars);
  cudaFree(c->aux_trace);
  cudaFree(c->splitk_ws);
  cudaFree(c->splitk_counters);
  cudaFree(c->reduce_ptrs_dev);
  cudaFree(c->signal_ptrs_dev);
  cudaFree(c->mailbox_ptrs_dev);
  for (int s = 0; s < 2; ++s) {
    cudaFree(c->h_img[s]);
    cudaFree(c->h_txt[s]);
    cudaFree(c->h_gimg[s]);
    cudaFree(c->h_gtxt[s]);
    if (c->ev_h2d[s]) cudaEventDestroy(c->ev_h2d[s]);
    if (c->ev_step[s]) cudaEventDestroy(c->ev_step[s]);
    if (c->ev_done[s]) cudaEventDestroy(c->ev_done[s]);
  }
  if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
  if (c->d2h_stream) cudaStreamDestroy(c->d2h_stream);
  if (c->h_pinned) cudaFreeHost(c->h_pinned);
  cudaFree(c->h_dimg);
  cudaFree(c->h_dtxt);
  if (c->dbg_host) cudaFreeHost(c->dbg_host);
  for (cudaEvent_t e : c->ev_loss) cudaEventDestroy(e);
  for (cudaEvent_t e : c->ev_grad) cudaEventDestroy(e);
  cudaGetLastError();
  delete c;
}

}  // namespace
