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
//   5 the retrieval-metric and per-sample-loss partials of forward #n are in place (siglip_request_metrics,
//     siglip_request_sample_losses)
constexpr int kFlagKinds = 6;
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
  int T;      // texts of the rank (B + its hard negatives)
  int Tmax;
  int R;      // images of the rank (B + its extra images)
  int Rmax;
  char host[56];
  int M;           // labels per set (siglip_ctx_create_labels; 0: none); inside the 64 bytes the host name had before
  int D_teacher;   // width of the gathered teacher text (0: none); inside the 64 bytes the host name had before
};

}  // namespace

struct siglip_ctx {
  int device = 0, rank = 0, world = 1, B = 0, D = 0, Bp = 0;
  int Bs[kMaxWorld] = {};                // per-rank batch (all equal to B unless created with siglip_ctx_create_uneven)
  int Bmax = 0;                          // max over ranks
  // text chunks (siglip_ctx_create_texts): rank p holds Ts[p] = Bs[p] + K_p texts, its B_p paired texts followed by K_p
  // hard negatives. Without extras Ts == Bs and everything below is what it was before they existed.
  int T = 0;                             // this rank's texts
  int Ts[kMaxWorld] = {};
  int Tmax = 0;                          // stride of every per-chunk text buffer is Tmax * D elements
  int Tp = 0;                            // columns of the sigma operands: Tmax rounded up to 256
  bool extras = false;                   // some rank has hard negatives (T_p != B_p)
  int toff[kMaxWorld + 1] = {};          // global index of every rank's first text (prefix sums of Ts)
  // extra images (siglip_ctx_create_extras): rank p holds Rs[p] = Bs[p] + E_p images, its B_p paired images followed by
  // E_p extras. Images never leave their rank. Without extra images Rs == Bs and everything below is what it was before
  // they existed.
  int R = 0;                             // this rank's images: rows of img / dimg
  int Rs[kMaxWorld] = {};
  int Rmax = 0;
  int Rp = 0;                            // rows of the sigma operands: Rmax rounded up to 256
  int Emax = 0;                          // max over ranks of the extra images (published ids per metrics step)
  bool ximg = false;                     // some rank has extra images (R_p != B_p)
  // this rank has extra images AND extra texts: the own chunk's positional diagonal row == col would also meet extra
  // rows and extra columns, so its loss kernel runs with own_chunk = 0 and takes every positive from ids instead (the
  // kIds instantiation, with row and column bounds; positional labels use iota ids)
  bool own_pos_ids = false;
  int extra_image_ids = 0;               // SIGLIP_OPT_EXTRA_IMAGE_IDS: the extra images carry ids (needs sample_ids)
  bool ximg_ids_set = false;             // siglip_set_extra_image_ids was called since the previous step
  int64_t* rids = nullptr;               // [R] ids of my images: B sample ids, then E extra-image ids (R > B only;
                                         // R == B: ids_in). Never exported
  int64_t* iota = nullptr;               // [max(R, T)] 0, 1, 2, ...: the positional labels of own_pos_ids
  int num_sms = 0;
  // options
  int cta_group = 2;
  int overlap_pull = 1;                  // pull the next text chunk inside the loss kernel
  int overlap_reduce = 1;                // fold the peers' dtxt contributions inside the gradient kernels
  int kernel_timing = 0;
  int stages_loss = 0, stages_grad = 0;  // 0 = kernel default
  int grad_tile_n = 0;                   // gradient kernel's column tiles: 0 = from the shape (grad_tile_cols), 128, 256
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
  int sample_ids = 0;                    // SIGLIP_OPT_SAMPLE_IDS: labels from per-sample ids (collective)
  bool ids_set = false;                  // siglip_set_sample_ids was called since the previous step
  int extra_text_ids = 0;                // SIGLIP_OPT_EXTRA_TEXT_IDS: the extras carry ids too (needs sample_ids)
  bool extra_ids_set = false;            // siglip_set_extra_text_ids was called since the previous step
  int sample_weights = 0;                // SIGLIP_OPT_SAMPLE_WEIGHTS: per-sample loss weights (collective)
  bool weights_set = false;              // siglip_set_sample_weights was called since the previous step
  int exclude_groups = 0;                // SIGLIP_OPT_EXCLUDE_GROUPS: same-group pairs are excluded (collective)
  bool groups_set = false;               // siglip_set_groups was called since the previous step
  bool ids_grp = false;                  // ids_in has its group halves (allocated when the mode is first turned on)
  // label sets (siglip_ctx_create_labels, SIGLIP_OPT_LABEL_SETS)
  int LM = 0;                            // labels per set M, 1 .. SIGLIP_MAX_LABELS (0: a context without label sets)
  int label_sets = 0;                    // SIGLIP_OPT_LABEL_SETS (collective)
  bool sets_set = false;                 // siglip_set_label_sets was called since the previous step
  int64_t* lrows = nullptr;              // [R][LM] the sets of my images: the paired ones, then the extras. Never exported
  // focal pair loss (SIGLIP_OPT_FOCAL): gamma and alpha are kernel parameters, kept until siglip_set_focal changes them
  int focal = 0;                         // SIGLIP_OPT_FOCAL (collective)
  bool focal_set = false;                // siglip_set_focal has been called
  float focal_gamma = 0.0f;
  float focal_alpha = -1.0f;             // < 0: no alpha
  // distillation (siglip_ctx_create_distill, SIGLIP_OPT_DISTILL)
  int DT = 0;                            // teacher width D_teacher (0: a context without a teacher)
  // siglip_ctx_create_distill_extras: distillation composes with per-sample losses, top-K, groups and label sets. A
  // siglip_ctx_create_distill context keeps refusing them, as it always has
  bool distill_opts = false;
  int distill = 0;                       // SIGLIP_OPT_DISTILL (collective)
  bool teacher_set = false;              // siglip_set_teacher was called since the previous step
  const void* t_img = nullptr;           // [B, DT] teacher images of the step (caller's buffer)
  const void* t_txt = nullptr;           // [B, DT] teacher texts of the step (caller's buffer)
  int t_f16 = 0;                         // teacher operands are fp16(x * 16)
  const float* t_tprime = nullptr;       // fp32 device scalars of the teacher
  const float* t_bias = nullptr;
  float t_lambda = 1.0f;
  __nv_bfloat16* ttxt_all = nullptr;     // [world][Bmax, DT] gathered teacher text (world > 1): behind the text weights in
                                         // the exported text allocation
  int off[kMaxWorld + 1] = {};           // global index of every rank's first image (prefix sums of Rs)
  // retrieval metrics (siglip_request_metrics), armed for the next step only
  bool metrics_armed = false;
  float* m_top1 = nullptr;
  int64_t* m_i2t = nullptr;
  int64_t* m_t2i = nullptr;
  unsigned long long* mkeys_step = nullptr;  // key block of the step being issued (null: no metrics this step)
  // per-sample losses (siglip_request_sample_losses), armed for the next step only
  bool losses_armed = false;
  float* l_img = nullptr;                // [R] image_loss output
  float* l_txt = nullptr;                // [T] text_loss output
  unsigned long long* lsum_step = nullptr;  // fixed-point block of the step being issued (null: no per-sample losses)
  // top-K retrieval (siglip_request_topk), armed for the next step only; K = 1 runs the metrics path
  bool topk_armed = false;
  int topk_k = 0;
  float* k_recall = nullptr;             // [2k]
  int64_t* k_i2t = nullptr;              // [ni, k] or null
  int64_t* k_t2i = nullptr;              // [nt, k] or null
  bool metrics_step = false;             // the step being issued writes the siglip_request_metrics outputs
  bool topk1_step = false;               // the step being issued writes K = 1 outputs from the metric keys
  bool topk_step = false;                // the step being issued fills the K > 1 lists (tk_cols / tk_rows of its parity)
  unsigned int topk_par = 0;             // ... whose parity is this
  // diagnostics, read from the environment once at context creation (see include/siglip_b200.h)
  bool dbg_no_gstore = false, dbg_no_cvt = false, dbg_loss_waitstats = false;
  // workspaces
  __nv_bfloat16* txt_all = nullptr;      // [world][Tmax, D] bf16; slot `rank` is what the peers pull (world > 1),
                                         // followed by ids_all in the same (IPC-exported) allocation
  int64_t* ids_all = nullptr;            // [world][ids_slot] ids (or label sets), then text groups, of every text chunk
                                         // (world > 1)
  int64_t* ids_in = nullptr;             // [ids_stride] this rank's ids for the next step: B sample ids
                                         // (siglip_set_sample_ids), then K extra-text ids (siglip_set_extra_text_ids);
                                         // once SIGLIP_OPT_EXCLUDE_GROUPS has been on, followed by [ids_stride] text
                                         // groups and [R] image groups (siglip_set_groups), laid out like a slot
  int ids_stride = 0;                    // Tmax rounded up to even: every slot is a whole number of 16-byte vectors.
                                         // Fixed at creation (options are set after the handle exchange)
  unsigned long long* mkeys[2] = {};     // per step parity: [world][Tmax] column argmax partials of every text chunk
                                         // over my images, then [Rmax] row keys, then [Emax] my extra-image ids (world > 1
                                         // under SIGLIP_OPT_EXTRA_IMAGE_IDS). world > 1: behind ids_all (exported)
  unsigned long long* lsum[2] = {};      // per step parity: [world][Tmax] column sums of every text chunk over my images,
                                         // [Rmax] row sums, then the same layout again for the poison bits
                                         // (lsum_block). world > 1: behind the gathered teacher text (exported)
  unsigned long long* tk_cols[2] = {};   // per step parity: [world][Tmax][kTopKMax] top-K column lists of every text
                                         // chunk over my images. world > 1: behind the loss partials (exported);
                                         // world == 1: allocated by the first siglip_request_topk
  unsigned long long* tk_rows[2] = {};   // per step parity: [Rmax][kTopKMax] row lists; allocated by the first request
  float* w_all = nullptr;                // [world][w_stride] text weights of every chunk (world > 1): behind the metric
                                         // keys in the exported allocation, sized at creation whatever the options
  float* w_in = nullptr;                 // [w_stride] my text weights, then [R] my image weights, clamped into [0, 1];
                                         // allocated by the first siglip_set_sample_weights
  int w_stride = 0;                      // Tmax rounded up to 4: every slot is a whole number of 16-byte vectors
  int sigma_budget_mib = 0;              // SIGLIP_OPT_SIGMA_BUDGET_MIB: bound of the sigma operands (0: none)
  int g_rows[kMaxWorld] = {};            // rows of each allocated sigma operand (Rp, or a panel height under a budget)
  __nv_bfloat16* G[kMaxWorld] = {};      // [Rp, Tp] sigma operands (fp16 bits x kGScale), diagonal zeroed, allocated on
                                         // first use: fused step 2 (own chunk + the chunk in flight), split API one per chunk
  __nv_bfloat16* img16 = nullptr;        // [R, D] fp16 (x kXScale) images: B operand of the dtxt contraction
  __nv_bfloat16* txt16[kMaxWorld] = {};  // [Tmax, D] fp16 (x kXScale) text chunks: B operand of dimg (same count as G)
  float* g_diag = nullptr;               // [Bp] fp32 positive-pair terms -sigma(-z_ii)
  float* slots = nullptr;                // [world][Tmax, D] fp32 dtxt contributions, slot c is for owner c (world > 1)
  float* dimg_acc = nullptr;             // [R, D] fp32 running dimg over the chunks (world > 1)
  float* dtxt_acc = nullptr;             // [T, D] fp32 running sum of the peers' contributions (world > 1)
  double* partials = nullptr;            // [num_sms][4]
  unsigned int* fin_counter = nullptr;   // ticket counter of the loss kernel's last-CTA finalisation
  unsigned int* flags = nullptr;         // [kFlagKinds][kMaxWorld]
  unsigned int* sync_words = nullptr;    // [kSyncWords] local tickets / flags
  float* loop_mailboxes = nullptr;       // loopback only: [world][2] stand-ins for the peers' (dt', dbias) mailboxes
  float* loop_zero = nullptr;            // loopback only: [world][Tmax, D] zeros standing in for the peers' contribution slots
  unsigned long long* loop_keys = nullptr;  // loopback only: [world][Tmax] the peers' column partials of my chunk
  unsigned long long* loop_lsums = nullptr;  // loopback only: [world] blocks standing in for the peers' loss partials
  unsigned long long* loop_topk = nullptr;   // loopback only: [world][Tmax][kTopKMax] the peers' column lists of my chunk
  int64_t* loop_xids = nullptr;          // loopback only: [world][Emax] the peers' published extra-image ids
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
  const unsigned long long** mkey_ptrs_dev = nullptr;  // [2][world] every rank's column partial of my chunk, per parity
  const unsigned long long** lsum_ptrs_dev = nullptr;  // [2][world] every rank's loss column partial of my chunk
  const unsigned long long** tk_ptrs_dev = nullptr;    // [2][world] every rank's top-K column lists of my chunk
  const int64_t** xid_ptrs_dev = nullptr;    // [2][world] every rank's published extra-image ids, per parity
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
    const bool peer = (code >= 5);   // 5 text pull, 6 helper wait, 7 fold, 8 last-fold flag, 9 scalar exchange, 10 metric partials, 1x aux jobs
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

// elements between consecutive text chunks of txt_all / slots / loop_zero (and the size of a txt16 copy)
inline size_t chunk_stride(const siglip_ctx* c) { return static_cast<size_t>(c->Tmax) * c->D; }

// Sample ids of text chunk `cidx` as the loss kernel reads them (null outside SIGLIP_OPT_SAMPLE_IDS): the caller's ids
// for the own chunk, the gathered copy for the others.
// Every slot of ids_all is [ids_stride] ids, then [ids_stride] text groups (SIGLIP_OPT_EXCLUDE_GROUPS), fixed at
// creation: the groups ride every copy of the ids, which then moves the whole slot. In a context with label sets the
// ids half is [ids_stride][M] set words (SIGLIP_OPT_LABEL_SETS: text l's set at l * M), the groups behind them.
inline size_t set_words(const siglip_ctx* c) {
  return static_cast<size_t>(c->ids_stride) * static_cast<size_t>(c->LM > 0 ? c->LM : 1);
}
inline size_t ids_slot(const siglip_ctx* c) { return set_words(c) + static_cast<size_t>(c->ids_stride); }
inline const int64_t* chunk_ids(const siglip_ctx* c, int cidx) {
  if (!c->sample_ids) return nullptr;
  return (cidx == c->rank) ? c->ids_in : c->ids_all + static_cast<size_t>(cidx) * ids_slot(c);
}
// Rank o's published ids slot, seen through its exported text allocation (they sit behind its [world][Tmax, D] text)
inline const int64_t* peer_ids(const siglip_ctx* c, int o) {
  return reinterpret_cast<const int64_t*>(c->peer_txt[o] + c->world * chunk_stride(c)) +
         static_cast<size_t>(o) * ids_slot(c);
}
// ---- excluded groups (SIGLIP_OPT_EXCLUDE_GROUPS) ----
// Text groups of chunk `cidx` as the loss kernel reads them (null outside the mode): the group half of my ids_in for
// the own chunk, of the gathered slot for the others. Image groups are local, behind my text groups: they never travel.
inline const int64_t* chunk_groups(const siglip_ctx* c, int cidx) {
  if (!c->exclude_groups) return nullptr;
  return ((cidx == c->rank) ? c->ids_in : c->ids_all + static_cast<size_t>(cidx) * ids_slot(c)) + set_words(c);
}
inline const int64_t* image_groups(const siglip_ctx* c) { return c->exclude_groups ? c->ids_in + ids_slot(c) : nullptr; }
// ---- label sets (SIGLIP_OPT_LABEL_SETS) ----
// Text sets of chunk `cidx` as the loss kernel reads them (null outside the mode): the set half of my ids_in for the
// own chunk, of the gathered slot for the others. Image sets are local (lrows): they never travel.
inline const int64_t* chunk_sets(const siglip_ctx* c, int cidx) {
  if (!c->label_sets) return nullptr;
  return (cidx == c->rank) ? c->ids_in : c->ids_all + static_cast<size_t>(cidx) * ids_slot(c);
}
// the ids copies of the exchange run in ids, groups or label-set mode; under the last two they move the whole slot
inline bool ids_travel(const siglip_ctx* c) { return c->sample_ids || c->exclude_groups || c->label_sets; }
// the sample ids of a rank (siglip_set_sample_ids)
inline size_t ids_bytes(const siglip_ctx* c, int rank) { return static_cast<size_t>(c->Bs[rank]) * sizeof(int64_t); }
// the ids of a text chunk as the exchange moves them: its paired texts', and under SIGLIP_OPT_EXTRA_TEXT_IDS its extras'
inline int chunk_id_count(const siglip_ctx* c, int rank) { return c->extra_text_ids ? c->Ts[rank] : c->Bs[rank]; }
inline size_t chunk_ids_bytes(const siglip_ctx* c, int rank) {
  return static_cast<size_t>(chunk_id_count(c, rank)) * sizeof(int64_t);
}
// bytes one ids copy of the exchange moves: the chunk's ids, or the whole slot (ids and text groups) under groups mode
inline size_t ids_copy_bytes(const siglip_ctx* c, int rank) {
  return (c->exclude_groups || c->label_sets) ? ids_slot(c) * sizeof(int64_t) : chunk_ids_bytes(c, rank);
}
// ids and weights of step s are given once: a step in ids / weights mode consumes them (all checked before anything is
// launched or consumed)
int take_ids(siglip_ctx* c) {
  if (c->losses_armed && c->distill && !c->distill_opts)
    return fail(SIGLIP_ERR_STATE, "per-sample losses are unavailable under SIGLIP_OPT_DISTILL on a "
                                  "siglip_ctx_create_distill context (siglip_ctx_create_distill_extras takes them)");
  if (c->topk_armed && c->distill && !c->distill_opts)
    return fail(SIGLIP_ERR_STATE, "top-K retrieval is unavailable under SIGLIP_OPT_DISTILL on a "
                                  "siglip_ctx_create_distill context (siglip_ctx_create_distill_extras takes it)");
  if (c->sample_ids && !c->ids_set)
    return fail(SIGLIP_ERR_STATE,
                "SIGLIP_OPT_SAMPLE_IDS is on but siglip_set_sample_ids was not called since the previous step");
  if (c->sample_ids && c->extra_text_ids && !c->extra_ids_set)
    return fail(SIGLIP_ERR_STATE,
                "SIGLIP_OPT_EXTRA_TEXT_IDS is on but siglip_set_extra_text_ids was not called since the previous step");
  if (c->sample_ids && c->extra_image_ids && !c->ximg_ids_set)
    return fail(SIGLIP_ERR_STATE,
                "SIGLIP_OPT_EXTRA_IMAGE_IDS is on but siglip_set_extra_image_ids was not called since the previous step");
  if (c->sample_weights && !c->weights_set)
    return fail(SIGLIP_ERR_STATE,
                "SIGLIP_OPT_SAMPLE_WEIGHTS is on but siglip_set_sample_weights was not called since the previous step");
  if (c->distill && !c->teacher_set)
    return fail(SIGLIP_ERR_STATE, "SIGLIP_OPT_DISTILL is on but siglip_set_teacher was not called since the previous step");
  if (c->exclude_groups && !c->groups_set)
    return fail(SIGLIP_ERR_STATE,
                "SIGLIP_OPT_EXCLUDE_GROUPS is on but siglip_set_groups was not called since the previous step");
  if (c->label_sets && !c->sets_set)
    return fail(SIGLIP_ERR_STATE,
                "SIGLIP_OPT_LABEL_SETS is on but siglip_set_label_sets was not called since the previous step");
  if (c->focal && !c->focal_set)
    return fail(SIGLIP_ERR_STATE, "SIGLIP_OPT_FOCAL is on but siglip_set_focal was never called");
  c->sets_set = false;
  c->groups_set = false;
  c->teacher_set = false;
  c->ids_set = false;
  c->extra_ids_set = false;
  c->ximg_ids_set = false;
  c->weights_set = false;
  return 0;
}

// ids of my images as the loss kernel reads them (ids mode): the sample ids, then the extra images' ids
inline const int64_t* row_ids(const siglip_ctx* c) { return c->rids != nullptr ? c->rids : c->ids_in; }
// rows that carry ids: the paired images, and under SIGLIP_OPT_EXTRA_IMAGE_IDS the extras too
inline int row_id_count(const siglip_ctx* c) { return c->extra_image_ids ? c->R : c->B; }

// ---- per-sample weights (SIGLIP_OPT_SAMPLE_WEIGHTS) ----
// Text weights of chunk `cidx` as the loss kernel reads them (null outside the mode): mine for the own chunk, the
// gathered copy for the others; the image weights are always mine (rows are local)
inline const float* chunk_weights(const siglip_ctx* c, int cidx) {
  if (!c->sample_weights) return nullptr;
  return (cidx == c->rank) ? c->w_in : c->w_all + static_cast<size_t>(cidx) * c->w_stride;
}
inline const float* image_weights(const siglip_ctx* c) { return c->sample_weights ? c->w_in + c->w_stride : nullptr; }
inline size_t chunk_weights_bytes(const siglip_ctx* c, int rank) {
  return static_cast<size_t>(c->Ts[rank]) * sizeof(float);
}
inline unsigned long long peer_timeout_ns(const siglip_ctx* c) {
  return static_cast<unsigned long long>(c->peer_timeout_ms) * 1000000ull;
}

// ---- retrieval metrics (siglip_request_metrics) ----
static_assert(siglip::kMetricsMaxWorld == kMaxWorld, "the finalisation kernel takes one batch offset per rank");
static_assert(siglip::kTopKMax == SIGLIP_TOPK_MAX, "the top-K lists have SIGLIP_TOPK_MAX slots");
// 64-bit words per step parity: [world][Tmax] column partials (the loss kernel writes one per text of the chunk; the
// finalisation reads the paired ones), then [Rmax] row keys, then [Emax] extra-image ids of this rank (published for the
// peers' t2i hit test under SIGLIP_OPT_EXTRA_IMAGE_IDS; [Emax][M] extra-image sets in a context with label sets).
// Without extra images: [Bmax] row keys and nothing behind.
inline size_t mkeys_block(const siglip_ctx* c) {
  return static_cast<size_t>(c->world) * c->Tmax + static_cast<size_t>(c->Rmax) +
         static_cast<size_t>(c->Emax) * static_cast<size_t>(c->LM > 0 ? c->LM : 1);
}
// offset of the published extra-image ids in a key block
inline size_t mkeys_xids(const siglip_ctx* c) { return static_cast<size_t>(c->world) * c->Tmax + c->Rmax; }
inline size_t mkeys_rows(const siglip_ctx* c) { return static_cast<size_t>(c->world) * c->Tmax; }
// words per peer of the loopback stand-ins of the published extra-image ids (or sets)
inline size_t loop_xids_stride(const siglip_ctx* c) {
  return static_cast<size_t>(c->Emax) * static_cast<size_t>(c->LM > 0 ? c->LM : 1);
}
// byte offset of the two key blocks in the exported text allocation: behind the gathered text and ids
inline size_t mkeys_offset(const siglip_ctx* c) {
  return chunk_stride(c) * c->world * sizeof(__nv_bfloat16) + static_cast<size_t>(c->world) * ids_slot(c) * sizeof(int64_t);
}
// byte offset of the text-weight slots in the exported text allocation: behind the two key blocks
inline size_t weights_offset(const siglip_ctx* c) {
  return mkeys_offset(c) + 2 * mkeys_block(c) * sizeof(unsigned long long);
}
// Rank o's published text-weight slot, seen through its exported text allocation
inline const float* peer_weights(const siglip_ctx* c, int o) {
  return reinterpret_cast<const float*>(reinterpret_cast<const char*>(c->peer_txt[o]) + weights_offset(c)) +
         static_cast<size_t>(o) * c->w_stride;
}
// ---- distillation (SIGLIP_OPT_DISTILL) ----
// elements between consecutive teacher text chunks of ttxt_all: a chunk holds all T texts of its rank, paired then
// extras, as the student's does (without extra texts T = B, the layout it had before extras could have a teacher)
inline size_t teacher_stride(const siglip_ctx* c) { return static_cast<size_t>(c->Tmax) * c->DT; }
inline size_t teacher_chunk_bytes(const siglip_ctx* c, int rank) {
  return static_cast<size_t>(c->Ts[rank]) * c->DT * sizeof(__nv_bfloat16);
}
// byte offset of the gathered teacher text in the exported text allocation: behind the text weights
inline size_t teacher_offset(const siglip_ctx* c) {
  return weights_offset(c) + static_cast<size_t>(c->world) * c->w_stride * sizeof(float);
}
// Rank o's published teacher text slot, seen through its exported text allocation
inline const __nv_bfloat16* peer_teacher(const siglip_ctx* c, int o) {
  return reinterpret_cast<const __nv_bfloat16*>(reinterpret_cast<const char*>(c->peer_txt[o]) + teacher_offset(c)) +
         static_cast<size_t>(o) * teacher_stride(c);
}
// teacher text of chunk `cidx` as the loss kernel reads it: the caller's for the own chunk, the gathered copy otherwise
inline const void* teacher_chunk(const siglip_ctx* c, int cidx) {
  return (cidx == c->rank) ? c->t_txt : static_cast<const void*>(c->ttxt_all + cidx * teacher_stride(c));
}

// ---- per-sample losses (siglip_request_sample_losses) ----
// 64-bit words from a fixed-point sum to its poison word: [world][Tmax] column sums (the loss kernel writes one per text
// of every chunk), then [Rmax] row sums
inline size_t lsum_half(const siglip_ctx* c) { return static_cast<size_t>(c->world) * c->Tmax + c->Rmax; }
// words per step parity: the sums, then the poison words in the same layout
inline size_t lsum_block(const siglip_ctx* c) { return 2 * lsum_half(c); }
inline size_t lsum_rows(const siglip_ctx* c) { return static_cast<size_t>(c->world) * c->Tmax; }
// byte offset of the two blocks in the exported text allocation: behind the gathered teacher text (which is empty
// without a teacher), so that no earlier offset moves
inline size_t lsum_offset(const siglip_ctx* c) {
  return teacher_offset(c) + teacher_stride(c) * c->world * sizeof(__nv_bfloat16);
}

// A step with per-sample losses starts: the block of the step's parity is zeroed by one memset. The block is written
// by the step's loss kernels and read by the peers after flag kind 5 of the step, like the metric keys, and
// double-buffered by parity for the same reason (DESIGN.md, "Per-sample losses").
int take_sample_losses(siglip_ctx* c, unsigned int s, cudaStream_t st) {
  c->lsum_step = nullptr;
  if (!c->losses_armed) return 0;
  c->losses_armed = false;
  c->lsum_step = c->lsum[s & 1u];
  CK(cudaMemsetAsync(c->lsum_step, 0, lsum_block(c) * sizeof(unsigned long long), st));
  c->launches++;
  return 0;
}
// After the step's last loss kernel (and the metrics finalisation, if armed): combine the column sums of my chunk
// (W > 1: with every rank's, after flag kind 5, which this kernel raises unless the metrics finalisation did) and
// decode both sides into the caller's buffers.
int finalize_sample_losses(siglip_ctx* c, unsigned int s, bool signal, cudaStream_t st) {
  if (c->lsum_step == nullptr) return 0;
  const int W = c->world;
  siglip::SampleLossArgs a;
  memset(&a, 0, sizeof(a));
  a.rows = c->lsum_step + lsum_rows(c);
  a.col_own = c->lsum_step + static_cast<size_t>(c->rank) * c->Tmax;
  a.poison = static_cast<long long>(lsum_half(c));
  a.R = c->R;
  a.T = c->T;
  a.rank = c->rank;
  a.world = W;
  a.signal = signal ? 1 : 0;
  a.image_loss = c->l_img;
  a.text_loss = c->l_txt;
  if (W > 1) {
    a.col_peers = c->lsum_ptrs_dev + static_cast<size_t>(s & 1u) * W;
    a.sig_ptrs = c->signal_ptrs_dev + 5 * W;
    a.flags_local = c->flags + 5 * kMaxWorld;
    a.value = s;
    a.timeout_ns = peer_timeout_ns(c);
  }
  a.dbg = c->dbg_dev;
  c->lsum_step = nullptr;
  CKI(siglip::launch_sample_loss_finalize(a, st));
  c->launches++;
  return 0;
}

// A metrics step starts (armed by siglip_request_metrics for this step only): the key block of the step's parity is
// zeroed, so that no max of an earlier step survives. Double-buffered by parity: a peer may still read my partials of
// step n in its finalisation while my step n + 1 writes; by step n + 2 that read is over (DESIGN.md, "In-batch
// retrieval metrics").
// A top-K request with K = 1 takes this path too (its outputs are the metric keys'), with or without a metrics request.
int take_metrics(siglip_ctx* c, unsigned int s, cudaStream_t st) {
  c->mkeys_step = nullptr;
  c->topk1_step = c->topk_armed && c->topk_k == 1;
  if (c->topk1_step) c->topk_armed = false;
  c->metrics_step = c->metrics_armed;
  if (!c->metrics_armed && !c->topk1_step) return 0;
  c->metrics_armed = false;
  c->mkeys_step = c->mkeys[s & 1u];
  CK(cudaMemsetAsync(c->mkeys_step, 0, mkeys_block(c) * sizeof(unsigned long long), st));
  c->launches++;
  if (c->world > 1 && c->sample_ids && c->extra_image_ids && c->R > c->B) {
    // my extra images' ids, for the peers whose texts an extra image of mine wins: read by their finalisation after
    // flag kind 5 of this step, reused two steps later like the keys
    CK(cudaMemcpyAsync(c->mkeys_step + mkeys_xids(c), c->rids + c->B,
                       static_cast<size_t>(c->R - c->B) * sizeof(int64_t), cudaMemcpyDeviceToDevice, st));
  }
  if (c->world > 1 && c->label_sets && c->R > c->B) {   // my extra images' sets, in the same words
    CK(cudaMemcpyAsync(c->mkeys_step + mkeys_xids(c), c->lrows + static_cast<size_t>(c->B) * c->LM,
                       static_cast<size_t>(c->R - c->B) * c->LM * sizeof(int64_t), cudaMemcpyDeviceToDevice, st));
  }
  return 0;
}
// The finalisation arguments of step s: batches, hit rules and flags (shared with the top-K finalisation)
void fill_metrics_args(const siglip_ctx* c, unsigned int s, siglip::MetricsArgs& a) {
  const int W = c->world;
  memset(&a, 0, sizeof(a));
  a.B = c->B;
  a.R = c->R;
  a.rank = c->rank;
  a.world = W;
  for (int p = 0; p <= W; ++p) {
    a.off[p] = c->off[p];
    a.toff[p] = c->toff[p];
  }
  for (int p = 0; p < W; ++p) a.bs[p] = c->Bs[p];
  a.T = c->T;
  if (c->sample_ids) {
    a.ids_own = c->ids_in;
    a.row_ids = row_ids(c);
    a.ids_all = c->ids_all;
    a.ids_stride = static_cast<int>(ids_slot(c));
    a.extra_ids = c->extra_text_ids;
    a.extra_image_ids = c->extra_image_ids;
    if (W > 1 && c->xid_ptrs_dev != nullptr) a.xids_peers = c->xid_ptrs_dev + static_cast<size_t>(s & 1u) * W;
  }
  if (W > 1) {
    a.sig_ptrs = c->signal_ptrs_dev + 5 * W;
    a.flags_local = c->flags + 5 * kMaxWorld;
    a.value = s;
    a.timeout_ns = peer_timeout_ns(c);
  }
  a.dbg = c->dbg_dev;
}
// The label-set hit rule of step s (SIGLIP_OPT_LABEL_SETS): my sets, the gathered text sets and the peers' published
// extra-image sets
void fill_label_set_args(const siglip_ctx* c, unsigned int s, siglip::LabelSetArgs& l) {
  memset(&l, 0, sizeof(l));
  l.row_sets = c->lrows;
  l.text_own = c->ids_in;
  l.text_all = c->ids_all;
  l.slot = static_cast<long long>(ids_slot(c));
  if (c->world > 1 && c->xid_ptrs_dev != nullptr)
    l.xsets_peers = c->xid_ptrs_dev + static_cast<size_t>(s & 1u) * c->world;
  l.m = c->LM;
}

// After the step's last loss kernel: combine the keys (W > 1: with every rank's partials of my chunk, flag kind 5) and
// write the indices and the top-1 rates.
int finalize_metrics(siglip_ctx* c, unsigned int s, cudaStream_t st) {
  if (c->mkeys_step == nullptr) return 0;
  siglip::MetricsArgs a;
  fill_metrics_args(c, s, a);
  a.row_keys = c->mkeys_step + mkeys_rows(c);
  a.col_own = c->mkeys_step + static_cast<size_t>(c->rank) * c->Tmax;
  if (c->world > 1) a.col_peers = c->mkey_ptrs_dev + static_cast<size_t>(s & 1u) * c->world;
  c->mkeys_step = nullptr;
  // once per set of outputs: siglip_request_metrics', then a K = 1 top-K request's (the same keys; a second raise of
  // flag kind 5 with the same value changes nothing)
  for (int out = 0; out < 2; ++out) {
    if (!(out == 0 ? c->metrics_step : c->topk1_step)) continue;
    a.top1 = out == 0 ? c->m_top1 : c->k_recall;
    a.i2t = out == 0 ? c->m_i2t : c->k_i2t;
    a.t2i = out == 0 ? c->m_t2i : c->k_t2i;
    if (c->label_sets) {
      siglip::LabelSetArgs l;
      fill_label_set_args(c, s, l);
      CKI(siglip::launch_metrics_finalize_labels(a, l, st));
    } else {
      CKI(siglip::launch_metrics_finalize(a, st));
    }
    c->launches++;
  }
  c->metrics_step = c->topk1_step = false;
  return 0;
}

// ---- top-K retrieval (siglip_request_topk, K > 1) ----
inline size_t topk_cols_words(const siglip_ctx* c) { return static_cast<size_t>(c->world) * c->Tmax * siglip::kTopKMax; }
inline size_t topk_rows_words(const siglip_ctx* c) { return static_cast<size_t>(c->Rmax) * siglip::kTopKMax; }
// byte offset of the two column-list blocks in the exported text allocation: behind the per-sample-loss partials
inline size_t topk_offset(const siglip_ctx* c) { return lsum_offset(c) + 2 * lsum_block(c) * sizeof(unsigned long long); }

// A top-K step starts: the lists of the step's parity are zeroed (two memsets). Written by the step's loss kernels and
// read by the peers after flag kind 5 of the step, double-buffered by parity like the metric keys.
int take_topk(siglip_ctx* c, unsigned int s, cudaStream_t st) {
  c->topk_step = false;
  if (!c->topk_armed) return 0;   // (K = 1 was taken by take_metrics)
  c->topk_armed = false;
  c->topk_step = true;
  c->topk_par = s & 1u;
  CK(cudaMemsetAsync(c->tk_cols[s & 1u], 0, topk_cols_words(c) * sizeof(unsigned long long), st));
  CK(cudaMemsetAsync(c->tk_rows[s & 1u], 0, topk_rows_words(c) * sizeof(unsigned long long), st));
  c->launches += 2;
  if (c->world > 1 && c->sample_ids && c->extra_image_ids && c->R > c->B) {
    // my extra images' ids for the peers' t2i hit test, where take_metrics publishes them (the same words, if both)
    CK(cudaMemcpyAsync(c->mkeys[s & 1u] + mkeys_xids(c), c->rids + c->B,
                       static_cast<size_t>(c->R - c->B) * sizeof(int64_t), cudaMemcpyDeviceToDevice, st));
  }
  if (c->world > 1 && c->label_sets && c->R > c->B) {   // my extra images' sets, as take_metrics publishes them
    CK(cudaMemcpyAsync(c->mkeys[s & 1u] + mkeys_xids(c), c->lrows + static_cast<size_t>(c->B) * c->LM,
                       static_cast<size_t>(c->R - c->B) * c->LM * sizeof(int64_t), cudaMemcpyDeviceToDevice, st));
  }
  return 0;
}

// After the metrics finalisation (if any): merge the column lists of my chunk (W > 1: with every rank's, after flag
// kind 5, which this kernel raises unless the metrics finalisation did), decode both sides and count the recalls.
int finalize_topk(siglip_ctx* c, unsigned int s, bool signal, cudaStream_t st) {
  if (!c->topk_step) return 0;
  const int W = c->world;
  siglip::TopKArgs a;
  memset(&a, 0, sizeof(a));
  fill_metrics_args(c, s, a.m);
  a.rows = c->tk_rows[s & 1u];
  a.col_own = c->tk_cols[s & 1u] + static_cast<size_t>(c->rank) * c->Tmax * siglip::kTopKMax;
  if (W > 1) a.col_peers = c->tk_ptrs_dev + static_cast<size_t>(s & 1u) * W;
  a.k = c->topk_k;
  a.signal = signal ? 1 : 0;
  a.recall = c->k_recall;
  a.i2t = c->k_i2t;
  a.t2i = c->k_t2i;
  c->topk_step = false;
  if (c->label_sets) {
    siglip::LabelSetArgs l;
    fill_label_set_args(c, s, l);
    CKI(siglip::launch_topk_finalize_labels(a, l, st));
  } else {
    CKI(siglip::launch_topk_finalize(a, st));
  }
  c->launches++;
  return 0;
}

// The step's detached outputs, after its last loss kernel: the metrics, then the top-K lists, then the per-sample
// losses; the first finalisation at W > 1 raises flag kind 5
int finalize_step_outputs(siglip_ctx* c, unsigned int s, cudaStream_t st) {
  const bool metrics = c->mkeys_step != nullptr;
  const bool topk = c->topk_step;
  int rc;
  if ((rc = finalize_metrics(c, s, st))) return rc;
  if ((rc = finalize_topk(c, s, !metrics, st))) return rc;
  return finalize_sample_losses(c, s, !metrics && !topk, st);
}

// Sigma operand + fp16 text copy number i, allocated on first use. The fused step needs two (own chunk, chunk in
// flight), the split forward / backward API one per text chunk (they all live from the forward to the backward).
// rows: rows of the operand (0: Rp, the whole batch; a panel height under SIGLIP_OPT_SIGMA_BUDGET_MIB). An operand of
// another height is released first.
void release_g(siglip_ctx* c, int i) {
  if (c->G[i] == nullptr) return;
  cudaFree(c->G[i]);
  cudaFree(c->txt16[i]);
  c->workspace_bytes -= static_cast<size_t>(c->g_rows[i]) * c->Tp * sizeof(__nv_bfloat16) +
                        chunk_stride(c) * sizeof(__nv_bfloat16);
  c->G[i] = nullptr;
  c->txt16[i] = nullptr;
  c->g_rows[i] = 0;
}

int ensure_g(siglip_ctx* c, int i, int rows = 0, cudaError_t* err = nullptr) {
  if (rows == 0) rows = c->Rp;
  if (c->G[i] != nullptr && c->g_rows[i] == rows) return 0;
  release_g(c, i);
  const size_t gbytes = static_cast<size_t>(rows) * c->Tp * sizeof(__nv_bfloat16);
  const size_t tbytes = chunk_stride(c) * sizeof(__nv_bfloat16);
  cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&c->G[i]), gbytes);
  if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&c->txt16[i]), tbytes);
  if (e != cudaSuccess) {
    cudaGetLastError();
    if (err != nullptr) *err = e;
    if (c->G[i]) cudaFree(c->G[i]);
    c->G[i] = nullptr;
    char buf[256];
    snprintf(buf, sizeof(buf),
             "sigma operand %d needs %.2f GiB more device memory (B = %d: %d x %d 16-bit per text chunk kept for the "
             "backward; siglip_fwd_bwd needs 2 of them, the split forward/backward API one per rank; "
             "SIGLIP_OPT_SIGMA_BUDGET_MIB bounds them by running siglip_fwd_bwd in row panels): %s",
             i, static_cast<double>(gbytes + tbytes) / (1024.0 * 1024.0 * 1024.0), c->Bmax, rows, c->Tp,
             cudaGetErrorString(e));
    return fail(SIGLIP_ERR_CUDA, buf);
  }
  c->g_rows[i] = rows;
  c->workspace_bytes += gbytes + tbytes;
  return 0;
}

// ---- row panels (SIGLIP_OPT_SIGMA_BUDGET_MIB) ----
// The sigma operands of a step under a budget: `nbuf` buffers of buf_rows x Tp 16-bit, the R rows of the rank scored
// in panels of `rows` (a multiple of the cluster's 128 x cluster_size rows; the last one may be shorter). A budget that
// holds nbuf whole [Rp, Tp] operands (or none set) gives the unbounded layout: one panel of R rows in Rp-row buffers.
// Depends on the budget, the shapes and the cluster configuration only, never on free memory.
struct Panels {
  int rows = 0;       // panel height (0: the budget is below one minimal panel)
  int n = 1;          // panels
  int buf_rows = 0;   // rows of each sigma buffer
};
Panels sigma_panels(int R, int Rp, int Tp, int nbuf, int unit, long long budget_mib) {
  Panels pn;
  const long long row_bytes = static_cast<long long>(nbuf) * Tp * static_cast<long long>(sizeof(__nv_bfloat16));
  const long long budget = budget_mib * 1024ll * 1024ll;
  if (budget_mib <= 0 || static_cast<long long>(Rp) * row_bytes <= budget) {
    pn.rows = R;
    pn.buf_rows = Rp;
    return pn;
  }
  const long long P = budget / row_bytes / unit * unit;   // < Rp here
  if (P == 0) return pn;
  pn.buf_rows = static_cast<int>(P);
  pn.rows = P < R ? static_cast<int>(P) : R;
  pn.n = ceil_div(R, pn.rows);
  return pn;
}
// bytes of the smallest budget that runs: nbuf buffers of one minimal panel
inline long long sigma_min_bytes(int Tp, int nbuf, int unit) {
  return static_cast<long long>(nbuf) * unit * Tp * static_cast<long long>(sizeof(__nv_bfloat16));
}
// sigma buffers of the fused step: the own chunk's (kept to the end) and the one in flight at W > 1, one at W = 1
inline int fused_buffers(const siglip_ctx* c) { return c->world > 1 ? 2 : 1; }
inline int panel_unit(const siglip_ctx* c) { return 128 * siglip::cluster_size(c->cta_group, c->mcast); }
int step_panels(siglip_ctx* c, int nbuf, Panels* out) {
  *out = sigma_panels(c->R, c->Rp, c->Tp, nbuf, panel_unit(c), c->sigma_budget_mib);
  if (out->rows == 0) {
    char buf[256];
    snprintf(buf, sizeof(buf),
             "SIGLIP_OPT_SIGMA_BUDGET_MIB = %d is below one minimal sigma panel: %d buffer(s) of %d x %d 16-bit need "
             "%.1f MiB",
             c->sigma_budget_mib, nbuf, panel_unit(c), c->Tp,
             static_cast<double>(sigma_min_bytes(c->Tp, nbuf, panel_unit(c))) / (1024.0 * 1024.0));
    return fail(SIGLIP_ERR_INVALID, buf);
  }
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

// Rows [r0, r0 + rows) of this rank scored against columns [c0, c0 + cols) of a text chunk: a row panel of
// SIGLIP_OPT_SIGMA_BUDGET_MIB (the default is the whole chunk). Every row- and column-indexed pointer of the launch is
// offset by the window's origin, so the kernels see a matrix of their own: the own chunk's positives sit at local
// row == local column only when r0 == c0.
struct Window {
  int r0 = 0, rows = -1;   // -1: all R rows
  int c0 = 0, cols = -1;   // -1: the columns from c0 to the end of the chunk
};

// The loss kernel over one text chunk (Bn rows, owner's batch): S = img @ txt_c^T on wgmma, fused
// scale/bias/log-sigmoid/reduce. save: also write the sigma operand G[gi] (+ g_diag on the own chunk); the fp16 copies
// the gradient kernel needs are auxiliary jobs built by the caller.
// cidx: owner rank of the chunk; col_ids: sample ids of the chunk (null = positional labels).
int run_loss_chunk(siglip_ctx* c, int gi, int cidx, bool own, bool first, const void* img, const __nv_bfloat16* txt_c,
                   int Bn, const int64_t* col_ids, const float* t_prime, const float* bias, bool save, const AuxList& aux,
                   const FinJob* fin, const EndSignal& end, cudaStream_t st, const Window& win = Window()) {
  const int cg = c->cta_group;
  int rc;
  const int gidx = save ? gi : 0;
  if (c->G[gidx] == nullptr && (rc = ensure_g(c, gidx))) return rc;
  const int r0 = win.r0, c0 = win.c0;
  const int M = win.rows < 0 ? c->R : win.rows;
  Bn = win.cols < 0 ? Bn - c0 : win.cols;   // from here on: the window's columns
  img = static_cast<const char*>(img) + static_cast<size_t>(r0) * c->D * sizeof(__nv_bfloat16);
  txt_c += static_cast<size_t>(c0) * c->D;
  __nv_bfloat16* G = c->G[gidx] + c0;
  CUtensorMap tmA, tmB, tmG;
  if ((rc = encode_operand(&tmA, img, M, c->D, c->D, 0, 128))) return rc;
  const int mc = c->mcast;
  if ((rc = encode_operand(&tmB, txt_c, Bn, c->D, c->D, 0, siglip::b_box_rows_kmajor(siglip::cluster_size(cg, mc)))))
    return rc;
  // store map of the sigma operand: [R, Bn] inside the padded [Rp, Tp] buffer, one 16-row x 32-column slab per TMA store
  // (a panel: [rows, cols] at column c0 of a buffer of panel height)
  const int g_rows = M < c->g_rows[gidx] ? M : c->g_rows[gidx];
  if ((rc = encode_bf16_2d(&tmG, G, (uint64_t)Bn, (uint64_t)g_rows, (uint64_t)c->Tp, 32, 16,
                           CU_TENSOR_MAP_SWIZZLE_64B)))
    return rc;
  KernelParams p;
  memset(&p, 0, sizeof(p));
  // distillation: the teacher's images and text chunk are the second operand pair (K = DT), same boxes as the student's
  CUtensorMap tmTA = tmA, tmTB = tmB;
  if (c->distill) {
    const __nv_bfloat16* t_img = static_cast<const __nv_bfloat16*>(c->t_img) + static_cast<size_t>(r0) * c->DT;
    const __nv_bfloat16* t_txt = static_cast<const __nv_bfloat16*>(teacher_chunk(c, cidx)) + static_cast<size_t>(c0) * c->DT;
    if ((rc = encode_operand(&tmTA, t_img, M, c->DT, c->DT, 0, 128))) return rc;
    if ((rc = encode_operand(&tmTB, t_txt, Bn, c->DT, c->DT, 0,
                             siglip::b_box_rows_kmajor(siglip::cluster_size(cg, mc)))))
      return rc;
    p.k_teacher = c->DT;
    p.teacher_f16 = c->t_f16;
    p.t_prime_T = c->t_tprime;
    p.bias_T = c->t_bias;
    p.distill_lambda = c->t_lambda;
  }
  p.nprob = 1;
  // fp32-input path: both operands are fp16(x * kXScale), the accumulator is kXScale^2 <img, txt>
  p.prob[0].ab_f16 = c->input_f16;
  p.s_scale = c->input_f16 ? 1.0f / (kXScale * kXScale) : 1.0f;
  // rows: my images, the paired ones and then the extras; the loss still divides by the paired batch
  p.prob[0].M = M;
  p.prob[0].N = Bn;
  p.prob[0].K = c->D;
  p.t_prime = t_prime;
  p.bias = bias;
  p.inv_b = 1.0f / static_cast<float>(c->B);
  p.G = G;
  p.ldg = c->Tp;
  p.g_diag = c->g_diag + r0;
  // the own chunk's positives are its first B columns (row == col < M); the hard negatives behind them never are. With
  // extra images and extra texts on this rank, row == col would also meet them: the own chunk then takes its positives
  // from ids, bounded to the first B rows and columns (iota ids for positional labels), and leaves g_diag alone
  p.own_chunk = (own && !c->own_pos_ids) ? 1 : 0;
  p.store_g = save ? 1 : 0;
  p.g_scale = kGScale;
  auto rest = [](int n, int o) { return n > o ? n - o : 0; };   // entries of an id list past a window's origin
  if (col_ids != nullptr) {
    p.row_ids = row_ids(c) + r0;
    p.col_ids = col_ids + c0;
    // the chunk's ids cover its paired texts, and under SIGLIP_OPT_EXTRA_TEXT_IDS its extras too
    p.col_pos_n = rest(chunk_id_count(c, cidx), c0);
    // the rows' ids cover the paired images, and under SIGLIP_OPT_EXTRA_IMAGE_IDS the extras too
    p.row_pos_n = rest(row_id_count(c), r0);
  } else if (own && c->own_pos_ids) {
    p.row_ids = c->iota + r0;
    p.col_ids = c->iota + c0;
    p.col_pos_n = rest(c->B, c0);
    p.row_pos_n = rest(c->B, r0);
  }
  if (c->sample_weights) {   // the kWeights instantiation: w_ij = image weight i x text weight j of the chunk
    p.row_w = image_weights(c) + r0;
    p.col_w = chunk_weights(c, cidx) + c0;
  }
  if (c->exclude_groups) {   // the kModeGroups kernel: same-group pairs that are not positives are excluded
    p.row_grp = image_groups(c) + r0;
    p.col_grp = chunk_groups(c, cidx) + c0;
    p.grp_rows = rest(c->R, r0);
  }
  if (c->label_sets) {   // the kModeLabels kernel: pairs whose sets share a label are positives too
    p.row_lab = c->lrows + static_cast<size_t>(r0) * c->LM;
    p.col_lab = chunk_sets(c, cidx) + static_cast<size_t>(c0) * c->LM;
    p.lab_m = c->LM;
  }
  if (c->focal) {   // the kModeFocal kernel: focal terms, every other option at run time
    p.focal = 1;
    p.focal_gamma = c->focal_gamma;
    p.focal_alpha = c->focal_alpha;
  }
  if (c->mkeys_step != nullptr) {   // a metrics step: the kMetrics instantiation reduces the argmax keys
    p.row_keys = c->mkeys_step + mkeys_rows(c) + r0;
    p.col_keys = c->mkeys_step + static_cast<size_t>(cidx) * c->Tmax + c0;
    p.row_off = c->off[c->rank] + r0;
    p.col_off = c->toff[cidx] + c0;
  }
  if (c->lsum_step != nullptr) {   // a per-sample-loss step: the kModeSampleLoss kernel adds the row / column sums
    p.sl_rows = c->lsum_step + lsum_rows(c) + r0;
    p.sl_cols = c->lsum_step + static_cast<size_t>(cidx) * c->Tmax + c0;
    p.sl_poison = static_cast<long long>(lsum_half(c));
  }
  if (c->topk_step) {   // a top-K step (K > 1): the kModeTopK kernel fills the row / column lists
    p.tk_rows = c->tk_rows[c->topk_par] + static_cast<size_t>(r0) * siglip::kTopKMax;
    p.tk_cols = c->tk_cols[c->topk_par] + (static_cast<size_t>(cidx) * c->Tmax + c0) * siglip::kTopKMax;
    p.tk_k = c->topk_k;
    p.row_off = c->off[c->rank] + r0;
    p.col_off = c->toff[cidx] + c0;
  }
  p.partials = c->partials;
  p.accumulate_partials = first ? 0 : 1;  // the first chunk of a forward overwrites every slot of the grid
  p.grid_n = c->Tmax;                     // ... and every chunk launches that same grid (see launch_gemm)
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
  CKI(siglip::launch_gemm(cg, siglip::kModeLoss, c->stages_loss, mc, siglip::kTileCols, &tmA, &tmB, &tmTA, &tmTB,
                          &tmG, p, c->num_sms, st));
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

// the fp16 image copy (B operand of the dtxt contraction)
void add_img_cvt_job(siglip_ctx* c, AuxList& aux, const void* img) {
  if (c->dbg_no_cvt) return;
  siglip::AuxJob& ji = aux.add(siglip::kAuxCvt);
  ji.src = reinterpret_cast<const uint4*>(img);
  ji.dst = reinterpret_cast<uint4*>(c->img16);
  ji.n16 = static_cast<unsigned long long>(c->R) * c->D * sizeof(__nv_bfloat16) / 16;
  ji.cvt_copy = c->input_f16;
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
  if (own) add_img_cvt_job(c, aux, img);
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
// Bn is the chunk's text count (its batch plus its hard negatives); the bracketed terms cover the first B rows only.
//
// Column-tile width of a gradient launch whose two problems have M0 and M1 rows (N = D both). A 256-column tile does
// the work of two 128-column ones in less time (one wgmma m64n256 instead of two m64n128 reading the A tile twice), but
// there are half as many tiles to spread over the clusters of the persistent grid. A launch lasts about (waves: tiles
// per cluster, rounded up) x (time of one tile), and a 256-column tile took 0.84 - 0.9 x the time of two 128-column
// ones on an H100 SXM (400 W, tools/tile_width_ab.py). So 256 when 2 x 0.9 x its waves <= the waves of 128-column
// tiles: B = 16384 with D = 768, 1024 or 1152, but not D <= 128, B = 16384 with D = 384 (4 waves against 6) nor
// B = 4096 with D = 768 (2 against 3). Split-K (SIGLIP_OPT_SPLIT_K) keeps its workspace of 128-column partials.
int grad_tile_cols(const siglip_ctx* c, int M0, int M1) {
  if (c->split_k != 0 && c->mcast == 1) return siglip::kTileCols;
  if (c->grad_tile_n != 0) return c->grad_tile_n;
  const int cs = siglip::cluster_size(c->cta_group, c->mcast);
  const long long units = c->num_sms / cs > 0 ? c->num_sms / cs : 1;
  auto waves = [&](int w) {
    const long long tiles =
        static_cast<long long>(ceil_div(M0, 128 * cs) + ceil_div(M1, 128 * cs)) * ceil_div(c->D, w);
    return (tiles + units - 1) / units;
  };
  return 18 * waves(siglip::kWideTileCols) <= 10 * waves(siglip::kTileCols) ? siglip::kWideTileCols : siglip::kTileCols;
}

// A row panel of the gradient launch (SIGLIP_OPT_SIGMA_BUDGET_MIB): the sigma panel of rows [r0, r0 + rows) in buffer
// gb, the chunk's fp16 text in txt16[tb]. dimg takes rows [r0, r0 + rows) (its positive-pair term too, on the own
// chunk); dtxt sums over the panel's rows, and takes the positive-pair term of all B rows only when fix_dtxt (the last
// own-chunk launch, after every panel's g_diag is written). The default is the whole chunk in buffer gi.
struct GradPanel {
  int gb = -1, tb = -1;   // -1: gi
  int r0 = 0, rows = -1;  // -1: all R rows
  bool fix_dtxt = true;
};

int run_grad_chunk(siglip_ctx* c, int gi, bool own, const void* img, const __nv_bfloat16* txt_own, int Bn,
                   const float* t_prime, const float* grad_out, const GradOut& o, const AuxList& aux,
                   const EndSignal& end, cudaStream_t st, const GradPanel& gp = GradPanel()) {
  const int cg = c->cta_group;
  const int gb = gp.gb < 0 ? gi : gp.gb, tb = gp.tb < 0 ? gi : gp.tb;
  const int r0 = gp.r0, M = gp.rows < 0 ? c->R : gp.rows;
  const int tile_n = grad_tile_cols(c, M, Bn);
  const int bk = siglip::b_box_k_mnmajor(siglip::cluster_size(cg, c->mcast), tile_n);
  CUtensorMap tmA0, tmB0, tmA1, tmB1;
  int rc;
  if (c->G[gb] == nullptr) return fail(SIGLIP_ERR_STATE, "gradient kernel without a saved sigma operand");
  // G is [R, Bn]: the MN-major map of the dtxt problem reads R k-rows of it and the image copy R rows; TMA fills the
  // boxes past R with zeros, so a partial last k block adds nothing (a panel: rows [r0, r0 + M) of both)
  if ((rc = encode_operand(&tmA0, c->G[gb], M, Bn, c->Tp, 0, 128))) return rc;
  if ((rc = encode_operand(&tmB0, c->txt16[tb], c->D, Bn, c->D, 1, 0, bk))) return rc;
  if ((rc = encode_operand(&tmA1, c->G[gb], Bn, M, c->Tp, 1, 0))) return rc;
  if ((rc = encode_operand(&tmB1, c->img16 + static_cast<size_t>(r0) * c->D, c->D, M, c->D, 1, 0, bk))) return rc;
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
    pr.fix_vec = (own && !c->own_pos_ids) ? c->g_diag : nullptr;   // own_pos_ids: the positives are in G
    pr.fix_f16 = c->saved_f16;
    pr.fix_mat_scale = c->saved_f16 ? 1.0f / kXScale : 1.0f;
  }
  const size_t row_off = static_cast<size_t>(r0) * c->D;   // dimg elements before the panel
  p.prob[0].M = M;
  p.prob[0].K = Bn;
  p.prob[0].a_mn = 0;
  p.prob[0].out = static_cast<char*>(o.dimg_out) + row_off * (o.dimg_bf16 ? sizeof(__nv_bfloat16) : sizeof(float));
  p.prob[0].out_bf16 = o.dimg_bf16 ? 1 : 0;
  p.prob[0].add_src = o.dimg_add != nullptr ? o.dimg_add + row_off : nullptr;
  p.prob[0].ld_add = c->D;
  if (p.prob[0].fix_vec != nullptr) p.prob[0].fix_vec += r0;
  p.prob[0].fix_mat = (own && !c->own_pos_ids) ? txt_own + row_off : nullptr;
  if (!gp.fix_dtxt) p.prob[1].fix_vec = nullptr;
  p.prob[1].M = Bn;
  p.prob[1].K = M;
  p.prob[1].a_mn = 1;
  p.prob[1].out = o.dtxt_out;
  p.prob[1].out_bf16 = o.dtxt_bf16 ? 1 : 0;
  p.prob[1].add_src = o.dtxt_add;
  p.prob[1].ld_add = c->D;
  p.prob[1].fix_mat = (own && !c->own_pos_ids) ? reinterpret_cast<const __nv_bfloat16*>(img) : nullptr;
  p.p1_wait_flag = o.dtxt_add_flag;
  p.p1_wait_value = o.dtxt_add_value;
  // g_diag and both fix matrices hold this rank's B rows; the dtxt rows of the own chunk's hard negatives (B .. Bn) and
  // the dimg rows of its extra images (B .. R) have no positive-pair term. A panel past row 0 has B - r0 of them and no
  // dtxt term (the caller's choice above): the field covers the dimg problem alone
  // (a chunk other than the own one has no positive-pair term at all)
  if (p.prob[1].fix_vec != nullptr && r0 != 0)
    return fail(SIGLIP_ERR_INVALID, "a gradient panel past row 0 cannot take the dtxt positive term");
  p.fix_rows = c->B > r0 ? c->B - r0 : 0;
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
  CKI(siglip::launch_gemm(cg, siglip::kModeOut, c->stages_grad, c->mcast, tile_n, &tmA0, &tmB0, &tmA1, &tmB1,
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
  j.n16 = static_cast<unsigned long long>(c->Ts[o]) * c->D * sizeof(__nv_bfloat16) / 16;
  j.wait_flags = c->flags + 0 * kMaxWorld + o;
  j.wait_n = 1;
  j.wait_value = s;
  j.site = 5;
  if (ids_travel(c)) {
    // the chunk's ids (and text groups) ride the same flag: the owner published them before its text signal, and
    // every CTA has observed that flag in the job above before it runs this one
    siglip::AuxJob& ji = aux.add(siglip::kAuxCopy);
    ji.src = reinterpret_cast<const uint4*>(peer_ids(c, o));
    ji.dst = reinterpret_cast<uint4*>(c->ids_all + static_cast<size_t>(o) * ids_slot(c));
    ji.n16 = (ids_copy_bytes(c, o) + 15) / 16;   // within the slot: ids_stride is even
  }
  if (c->sample_weights) {
    // the chunk's text weights ride the same flag, like its ids
    siglip::AuxJob& jw = aux.add(siglip::kAuxCopy);
    jw.src = reinterpret_cast<const uint4*>(peer_weights(c, o));
    jw.dst = reinterpret_cast<uint4*>(c->w_all + static_cast<size_t>(o) * c->w_stride);
    jw.n16 = (chunk_weights_bytes(c, o) + 15) / 16;   // within the slot: w_stride is a multiple of 4
  }
  if (c->distill) {
    // the chunk's teacher text rides the same flag, like its ids
    siglip::AuxJob& jt = aux.add(siglip::kAuxCopy);
    jt.src = reinterpret_cast<const uint4*>(peer_teacher(c, o));
    jt.dst = reinterpret_cast<uint4*>(c->ttxt_all + o * teacher_stride(c));
    jt.n16 = teacher_chunk_bytes(c, o) / 16;   // DT % 8 == 0
  }
}

// publish job of my teacher text (L0 of the fused step), the twin of the ids publish job below
void add_teacher_publish_job(siglip_ctx* c, AuxList& aux, unsigned int s) {
  siglip::AuxJob& j = aux.add(siglip::kAuxCopy);
  j.src = reinterpret_cast<const uint4*>(c->t_txt);
  j.dst = reinterpret_cast<uint4*>(c->ttxt_all + c->rank * teacher_stride(c));
  j.n16 = teacher_chunk_bytes(c, c->rank) / 16;
  j.wait_flags = c->flags + 2 * kMaxWorld;
  j.wait_n = c->world;
  j.wait_value = s - 1;
  j.site = 11;
}

// publish job of my text weights (L0 of the fused step), the twin of the ids publish job below
void add_weights_publish_job(siglip_ctx* c, AuxList& aux, unsigned int s) {
  siglip::AuxJob& j = aux.add(siglip::kAuxCopy);
  j.src = reinterpret_cast<const uint4*>(c->w_in);
  j.dst = reinterpret_cast<uint4*>(c->w_all + static_cast<size_t>(c->rank) * c->w_stride);
  j.n16 = (chunk_weights_bytes(c, c->rank) + 15) / 16;
  j.wait_flags = c->flags + 2 * kMaxWorld;
  j.wait_n = c->world;
  j.wait_value = s - 1;
  j.site = 11;
}

// publish job of my ids (L0 of the fused step): same flag-2 wait as the text publish job that must follow it in the
// same launch, whose end-of-job signal then covers both copies
void add_ids_publish_job(siglip_ctx* c, AuxList& aux, unsigned int s) {
  siglip::AuxJob& j = aux.add(siglip::kAuxCopy);
  j.src = reinterpret_cast<const uint4*>(c->ids_in);
  j.dst = reinterpret_cast<uint4*>(c->ids_all + static_cast<size_t>(c->rank) * ids_slot(c));
  j.n16 = (ids_copy_bytes(c, c->rank) + 15) / 16;
  j.wait_flags = c->flags + 2 * kMaxWorld;
  j.wait_n = c->world;
  j.wait_value = s - 1;
  j.site = 11;
}

// the same publishes (ids, text weights) as stream copies (split forward, helper-kernel variant of the fused step)
int copy_own_chunk_data(siglip_ctx* c, cudaStream_t st) {
  if (ids_travel(c))
    CK(cudaMemcpyAsync(c->ids_all + static_cast<size_t>(c->rank) * ids_slot(c), c->ids_in,
                       ids_copy_bytes(c, c->rank), cudaMemcpyDeviceToDevice, st));
  if (c->sample_weights)
    CK(cudaMemcpyAsync(c->w_all + static_cast<size_t>(c->rank) * c->w_stride, c->w_in, chunk_weights_bytes(c, c->rank),
                       cudaMemcpyDeviceToDevice, st));
  if (c->distill)
    CK(cudaMemcpyAsync(c->ttxt_all + c->rank * teacher_stride(c), c->t_txt, teacher_chunk_bytes(c, c->rank),
                       cudaMemcpyDeviceToDevice, st));
  return 0;
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
  if (c->sigma_budget_mib > 0) {
    Panels pn;
    if (save) {
      // the split API keeps one whole operand per chunk until the backward: no panels
      pn = sigma_panels(c->R, c->Rp, c->Tp, c->world, panel_unit(c), c->sigma_budget_mib);
      if (pn.n > 1 || pn.buf_rows != c->Rp) {
        char buf[320];
        snprintf(buf, sizeof(buf),
                 "siglip_forward with save_for_backward keeps %d sigma operands of %d x %d 16-bit (%.2f GiB) until "
                 "the backward, more than SIGLIP_OPT_SIGMA_BUDGET_MIB = %d: use siglip_fwd_bwd, which runs in row panels",
                 c->world, c->Rp, c->Tp,
                 static_cast<double>(c->world) * c->Rp * c->Tp * sizeof(__nv_bfloat16) / (1024.0 * 1024.0 * 1024.0),
                 c->sigma_budget_mib);
        return fail(SIGLIP_ERR_STATE, buf);
      }
    } else if (c->G[0] == nullptr) {
      // a forward without save writes no sigma: one panel-sized buffer backs the (unused) store map
      if ((rc = step_panels(c, 1, &pn))) return rc;
      CK(cudaSetDevice(c->device));
      if ((rc = ensure_g(c, 0, pn.buf_rows))) return rc;
    }
  }
  if ((rc = take_ids(c))) return rc;
  CK(cudaSetDevice(c->device));
  const int W = c->world, r = c->rank;
  const size_t stride = chunk_stride(c);
  const unsigned int s = ++c->n_fwd;
  if ((rc = take_metrics(c, s, st))) return rc;
  if ((rc = take_sample_losses(c, s, st))) return rc;
  if ((rc = take_topk(c, s, st))) return rc;
  // the saved state is being overwritten (a forward without save still replaces my gathered text slot, which the
  // backward of a multi-rank job reads for the positive-pair term); valid again once a saving forward is enqueued
  if (save || c->world > 1) c->gen = 0;

  const __nv_bfloat16* own_txt = reinterpret_cast<const __nv_bfloat16*>(txt);
  if (W > 1) {
    // peers must have finished pulling my text slot in their previous forward before I overwrite it
    if ((rc = wait_peers(c, 2, s - 1, st))) return rc;
    CK(cudaMemcpyAsync(c->txt_all + r * stride, txt, static_cast<size_t>(c->T) * c->D * sizeof(__nv_bfloat16),
                       cudaMemcpyDeviceToDevice, st));
    if ((rc = copy_own_chunk_data(c, st))) return rc;   // before the signal, which covers it
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
    if (save) add_cvt_jobs(c, aux, k, k == 0, img, txt_c, c->Ts[cidx]);
    if (k + 1 < W) {
      const int nxt = step_owner(c, r, k + 1);
      if (c->overlap_pull) {
        add_pull_job(c, aux, nxt, s);
      } else {
        // un-overlapped variant (A/B measurements): wait + copy as separate stream operations
        if ((rc = wait_one(c, 0, nxt, s, st))) return rc;
        CK(cudaMemcpyAsync(c->txt_all + nxt * stride, c->peer_txt[nxt] + nxt * stride,
                           static_cast<size_t>(c->Ts[nxt]) * c->D * sizeof(__nv_bfloat16), cudaMemcpyDefault, st));
        if (ids_travel(c))
          CK(cudaMemcpyAsync(c->ids_all + static_cast<size_t>(nxt) * ids_slot(c), peer_ids(c, nxt),
                             ids_copy_bytes(c, nxt), cudaMemcpyDefault, st));
        if (c->sample_weights)
          CK(cudaMemcpyAsync(c->w_all + static_cast<size_t>(nxt) * c->w_stride, peer_weights(c, nxt),
                             chunk_weights_bytes(c, nxt), cudaMemcpyDefault, st));
        if (c->distill)
          CK(cudaMemcpyAsync(c->ttxt_all + nxt * teacher_stride(c), peer_teacher(c, nxt), teacher_chunk_bytes(c, nxt),
                             cudaMemcpyDefault, st));
      }
    }
    if ((rc = run_loss_chunk(c, k, cidx, k == 0, k == 0, img, txt_c, c->Ts[cidx], chunk_ids(c, cidx), t_prime, bias, save,
                             aux, (k == W - 1) ? &fin : nullptr, EndSignal(), st)))
      return rc;
  }
  if (W > 1) {
    if ((rc = signal_peers(c, 2, s, st))) return rc;
  }
  if ((rc = finalize_step_outputs(c, s, st))) return rc;
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
      f.n16 = static_cast<unsigned long long>(c->T) * c->D * sizeof(float) / 16;
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
    if ((rc = run_grad_chunk(c, k, k == 0, img, own_txt, c->Ts[cidx], t_prime, grad_out, o, aux, EndSignal(), st)))
      return rc;
    if (W > 1 && (!last || !c->overlap_reduce)) {
      if ((rc = signal_peers(c, 1, base + static_cast<unsigned int>(j), st))) return rc;
    }
  }
  if (W > 1) {
    if (c->overlap_reduce) {
      // dtxt = (sum of the W-1 remote contributions, already local) + my own contribution: a local add
      CKI(siglip::launch_reduce_slots(dtxt, c->grad_bf16, c->final_ptrs_dev, 2, static_cast<size_t>(c->T) * c->D,
                                      c->num_sms, st));
    } else {
      if ((rc = wait_peers(c, 1, base + static_cast<unsigned int>(W), st))) return rc;
      CKI(siglip::launch_reduce_slots(dtxt, c->grad_bf16, c->reduce_ptrs_dev, W, static_cast<size_t>(c->T) * c->D,
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
//
// Under SIGLIP_OPT_SIGMA_BUDGET_MIB the rows are scored in np panels of P rows (DESIGN.md, "Row panels"): every sigma
// operand holds one panel, and each chunk runs L G per panel (index k.p below). Panel 0 of the own chunk keeps the
// role of L0 / G0, so the exchange keeps its shape:
//   W > 1:  L0.0  [L0.p G0.p]p=np-1..1  [L1.p G1.p]p=0..np-1  ...  [L(W-1).p G(W-1).p]  G0.0
//   W = 1:        [L0.p G0.p]p=np-1..1  L0.0 G0.0          (one buffer: nothing is in flight)
// Flag 1 of a remote chunk is raised by its last panel's gradient launch; its earlier panels add into the slot. The
// own panels past 0 sum their dtxt into a local partial (slot `rank`, which no peer reads in this step, or dtxt_acc at
// W = 1) that enters the first fold, and G0.0 adds the positive-pair term of all B rows to dtxt. With one panel the
// launches are exactly the unbounded step's.
// ---------------------------------------------------------------------------------------------------------------
int fused_impl(siglip_ctx* c, const void* img, const void* txt, const float* t_prime, const float* bias, float* loss,
               const float* grad_out, void* dimg, void* dtxt, float* dt_prime, float* dbias, cudaStream_t st) {
  int rc;
  if ((rc = check_call(c, img, txt, t_prime, st))) return rc;
  if (bias == nullptr || loss == nullptr || dimg == nullptr || dtxt == nullptr)
    return fail(SIGLIP_ERR_INVALID, "null argument");
  if ((rc = check_dbg(c, "siglip_fwd_bwd (previous launch)"))) return rc;
  Panels pn;
  if ((rc = step_panels(c, fused_buffers(c), &pn))) return rc;
  if ((rc = take_ids(c))) return rc;
  CK(cudaSetDevice(c->device));
  const int W = c->world, r = c->rank;
  const int np = pn.n, P = pn.rows;
  auto prow = [&](int p) { return c->R - p * P < P ? c->R - p * P : P; };
  const size_t stride = chunk_stride(c);
  const unsigned int s = ++c->n_fwd;
  const unsigned int n = ++c->n_bwd;
  const unsigned int base = (n - 1) * static_cast<unsigned int>(W);
  const bool ik = c->inkernel_sync != 0;
  if ((rc = take_metrics(c, s, st))) return rc;
  if ((rc = take_sample_losses(c, s, st))) return rc;
  if ((rc = take_topk(c, s, st))) return rc;
  c->gen = 0;                       // the sigma operands of a split forward (if any) are overwritten
  c->saved_f16 = c->input_f16;
  if ((rc = ensure_g(c, 0, pn.buf_rows))) return rc;
  if (W > 1 && (rc = ensure_g(c, 1, pn.buf_rows))) return rc;
  if (W == 1 && np > 1 && c->dtxt_acc == nullptr) {
    const size_t bytes = static_cast<size_t>(c->T) * c->D * sizeof(float);
    CK(cudaMalloc(reinterpret_cast<void**>(&c->dtxt_acc), bytes));
    c->workspace_bytes += bytes;
  }
  // dtxt of the own panels past 0 (fp32, [T, D]), added to the fold chain (W > 1) or by G0.0 (W = 1)
  float* own_part = (np > 1) ? ((W > 1) ? c->slots + r * stride : c->dtxt_acc) : nullptr;
  const __nv_bfloat16* own_txt = reinterpret_cast<const __nv_bfloat16*>(txt);
  const size_t own_bytes = static_cast<size_t>(c->T) * c->D * sizeof(__nv_bfloat16);
  FinJob fin;
  fin.loss = loss;
  fin.dt_prime = c->scalars + kSavedScalars;
  fin.dbias = c->scalars + kSavedScalars + 1;
  // With ids and weights, L0 would carry 9 jobs (3 publishes, 2 conversions, the flag-3 wait, 3 pulls) of
  // kMaxAuxJobs = 8: the image conversion then runs in L1 instead (its first reader is G1, behind L1).
  // (Groups mode runs the same ids jobs, so it counts as ids here.)
  const bool img_cvt_in_l1 = W > 1 && ik && ((ids_travel(c) && c->sample_weights) || c->distill);
  // Distillation adds a teacher publish and a teacher pull to L0 (up to 8 jobs with ids and weights): the own text's
  // conversion and the flag-3 wait move to L1 as well. G0, their first consumer, and G1 run behind L1.
  const bool l0_work_in_l1 = W > 1 && ik && c->distill;
  // with panels, those jobs go to the launch behind L0.0, the first own panel's loss kernel (G0.p reads them)
  const bool moved_to_l1 = np == 1;

  // ---- L0: own chunk. Its auxiliary warps also publish my text to the peers and start the first pull ----
  if (W > 1 || np == 1) {
    AuxList aux;
    if (W > 1) {
      if (ik) {
        // my gathered slot is what the peers pull: they must be done with the previous forward's copy (flag 2),
        // then "text of forward s in place" (flag 0) goes to every rank once all CTAs have copied their share. My
        // ids (sample-id mode) and text weights (weights mode) are copied by jobs before it: each CTA finishes them
        // before the text job's ticket, so the same signal covers them.
        if (ids_travel(c)) add_ids_publish_job(c, aux, s);
        if (c->sample_weights) add_weights_publish_job(c, aux, s);
        if (c->distill) add_teacher_publish_job(c, aux, s);
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
        if ((rc = copy_own_chunk_data(c, st))) return rc;
        if ((rc = signal_peers(c, 0, s, st))) return rc;
      }
    }
    if (!l0_work_in_l1) add_cvt_jobs(c, aux, 0, !img_cvt_in_l1, img, own_txt, c->T);
    if (W > 1) {
      if (ik && l0_work_in_l1) {
        // the flag-3 wait runs in L1 (before G1 all the same)
      } else if (ik) {
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
    Window w0;
    w0.rows = prow(0);
    if ((rc = run_loss_chunk(c, 0, r, true, true, img, own_txt, c->T, chunk_ids(c, r), t_prime, bias, true, aux,
                             (W == 1) ? &fin : nullptr, EndSignal(), st, w0)))
      return rc;
  }
  if (W > 1) own_txt = c->txt_all + r * stride;   // the copy the peers see (same bytes)
  // ---- own panels past 0: L0.p G0.p in the buffer of the chunks in flight (W = 1: the only buffer) ----
  for (int p = np - 1; p >= 1; --p) {
    const int p0 = p * P, rows = prow(p), gb = (W > 1) ? 1 : 0;
    const bool first_launch = (W == 1 && p == np - 1);
    AuxList aux;
    if (first_launch) {
      add_cvt_jobs(c, aux, 0, true, img, own_txt, c->T);
      // A loss launch's grid follows its panel's row tiles, and this shortest panel runs first: its CTAs overwrite
      // their partial slots only. L0.0, the largest panel, runs last and adds into every slot, so the slots past this
      // launch's grid would carry the previous step's sums into this step's loss, dt' and dbias.
      CK(cudaMemsetAsync(c->partials, 0, static_cast<size_t>(c->num_sms) * 4 * sizeof(double), st));
      c->launches++;
    }
    if (W > 1 && p == np - 1) {
      if (img_cvt_in_l1) add_img_cvt_job(c, aux, img);
      if (l0_work_in_l1) {
        add_cvt_jobs(c, aux, 0, false, img, reinterpret_cast<const __nv_bfloat16*>(txt), c->T);
        siglip::AuxJob& w3 = aux.add(siglip::kAuxWaitOnly);
        w3.wait_flags = c->flags + 3 * kMaxWorld;
        w3.wait_n = W;
        w3.wait_value = n - 1;
        w3.site = 13;
      }
    }
    // The panel's positives sit in columns [p0, p0 + rows): scored with the own-chunk diagonal in a window that starts
    // at column p0, the columns before it in a second launch without one. iota ids (own_pos_ids) and rows past B need
    // one launch.
    const bool own_rows = p0 < c->B;
    Window w;
    w.r0 = p0;
    w.rows = rows;
    if (own_rows && !c->own_pos_ids) {
      w.c0 = p0;
      if ((rc = run_loss_chunk(c, gb, r, true, first_launch, img, own_txt, c->T, chunk_ids(c, r), t_prime, bias, true,
                               aux, nullptr, EndSignal(), st, w)))
        return rc;
      w.c0 = 0;
      w.cols = p0;
      if ((rc = run_loss_chunk(c, gb, r, false, false, img, own_txt, c->T, chunk_ids(c, r), t_prime, bias, true,
                               AuxList(), nullptr, EndSignal(), st, w)))
        return rc;
    } else if ((rc = run_loss_chunk(c, gb, r, own_rows, first_launch, img, own_txt, c->T, chunk_ids(c, r), t_prime,
                                    bias, true, aux, nullptr, EndSignal(), st, w))) {
      return rc;
    }
    GradOut o;
    o.dimg_out = (W > 1) ? static_cast<void*>(c->dimg_acc) : dimg;   // W = 1: these rows are final
    o.dimg_bf16 = W == 1 && c->grad_bf16;
    o.dtxt_out = own_part;
    o.dtxt_add = (p == np - 1) ? nullptr : own_part;
    GradPanel gp;
    gp.gb = gb;
    gp.tb = 0;
    gp.r0 = p0;
    gp.rows = rows;
    gp.fix_dtxt = false;
    if ((rc = run_grad_chunk(c, gb, true, img, own_txt, c->T, t_prime, grad_out, o, AuxList(), EndSignal(), st, gp)))
      return rc;
  }
  // ---- remote chunks: L_k then G_k (gradient slot j = k) ----
  for (int k = 1; k < W; ++k) {
    const int cidx = step_owner(c, r, k);
    const __nv_bfloat16* txt_c = c->txt_all + cidx * stride;
   for (int p = 0; p < np; ++p) {
    const int p0 = p * P;
    {
      AuxList aux;
      if (p == 0) add_cvt_jobs(c, aux, 1, k == 1 && img_cvt_in_l1 && moved_to_l1, img, txt_c, c->Ts[cidx]);
      if (p == 0 && k == 1 && l0_work_in_l1 && moved_to_l1) {
        add_cvt_jobs(c, aux, 0, false, img, reinterpret_cast<const __nv_bfloat16*>(txt), c->T);
        siglip::AuxJob& w3 = aux.add(siglip::kAuxWaitOnly);
        w3.wait_flags = c->flags + 3 * kMaxWorld;
        w3.wait_n = W;
        w3.wait_value = n - 1;
        w3.site = 13;
      }
      if (p == 0 && k + 1 < W) add_pull_job(c, aux, step_owner(c, r, k + 1), s);
      const bool lastL = (k == W - 1) && (p == np - 1);
      EndSignal end = (lastL && ik) ? end_signal(c, 2, s) : EndSignal();   // "I have pulled everyone's text"
      Window w;
      w.r0 = p0;
      w.rows = prow(p);
      if ((rc = run_loss_chunk(c, 1, cidx, false, false, img, txt_c, c->Ts[cidx], chunk_ids(c, cidx), t_prime, bias, true,
                               aux, lastL ? &fin : nullptr, end, st, w)))
        return rc;
      if (lastL && !ik && (rc = signal_peers(c, 2, s, st))) return rc;
    }
    const int j = k;
    // dimg rows of a panel past 0 were started by their own panel, and the last chunk finishes them
    const bool rows_final = p > 0 && k == W - 1;
    GradOut o;
    o.dimg_add = (j > 1 || p > 0) ? c->dimg_acc : nullptr;
    o.dimg_out = rows_final ? dimg : static_cast<void*>(c->dimg_acc);
    o.dimg_bf16 = rows_final && c->grad_bf16;
    o.dtxt_out = c->slots + cidx * stride;
    o.dtxt_add = (p > 0) ? c->slots + cidx * stride : nullptr;   // the chunk's earlier panels
    AuxList aux;
    if (j >= 2 && p == 0) {
      const int pr = ((r - step_offset(c, j - 1)) % W + W) % W;
      siglip::AuxJob& f = aux.add(siglip::kAuxFold);
      f.src = reinterpret_cast<const uint4*>(c->peer_slots[pr] + r * stride);
      f.src2 = reinterpret_cast<const uint4*>((j == 2) ? own_part : c->dtxt_acc);
      f.dst = reinterpret_cast<uint4*>(c->dtxt_acc);
      f.n16 = static_cast<unsigned long long>(c->T) * c->D * sizeof(float) / 16;
      f.wait_flags = c->flags + 1 * kMaxWorld + pr;
      f.wait_n = 1;
      f.wait_value = base + static_cast<unsigned int>(j - 1);
      f.site = 7;
    }
    // "my contribution to owner cidx is complete": its last panel only
    const bool lastG = p == np - 1;
    EndSignal end = (ik && lastG) ? end_signal(c, 1, base + static_cast<unsigned int>(j)) : EndSignal();
    GradPanel gp;
    gp.r0 = p0;
    gp.rows = prow(p);
    if ((rc = run_grad_chunk(c, 1, false, img, own_txt, c->Ts[cidx], t_prime, grad_out, o, aux, end, st, gp)))
      return rc;
    if (!ik && lastG && (rc = signal_peers(c, 1, base + static_cast<unsigned int>(j), st))) return rc;
   }
  }
  // ---- W = 1 with panels: L0.0 last, in the buffer G0.0 reads ----
  if (W == 1 && np > 1) {
    Window w0;
    w0.rows = prow(0);
    if ((rc = run_loss_chunk(c, 0, r, true, false, img, own_txt, c->T, chunk_ids(c, r), t_prime, bias, true, AuxList(),
                             &fin, EndSignal(), st, w0)))
      return rc;
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
      f.src2 = reinterpret_cast<const uint4*>((W == 2) ? own_part : c->dtxt_acc);
      f.dst = reinterpret_cast<uint4*>(c->dtxt_acc);
      f.n16 = static_cast<unsigned long long>(c->T) * c->D * sizeof(float) / 16;
      f.wait_flags = c->flags + 1 * kMaxWorld + pr;
      f.wait_n = 1;
      f.wait_value = base + static_cast<unsigned int>(W - 1);
      f.site = 7;
      f.done_flag = c->sync_words + kSyncFoldDone;
      f.done_value = n;
      o.dtxt_add = c->dtxt_acc;
      o.dtxt_add_flag = c->sync_words + kSyncFoldDone;
      o.dtxt_add_value = n;
    } else if (np > 1) {
      o.dtxt_add = own_part;   // W = 1: the own panels past 0, written by the launches before this one
    }
    const bool scalars_here = !(W > 1 && c->sync_scalar_grads);
    o.sc_dt_prime = scalars_here ? dt_prime : nullptr;
    o.sc_dbias = scalars_here ? dbias : nullptr;
    EndSignal end = (W > 1 && ik) ? end_signal(c, 3, n) : EndSignal();   // "I have read everyone's contributions"
    GradPanel gp;
    gp.rows = prow(0);
    if ((rc = run_grad_chunk(c, 0, true, img, own_txt, c->T, t_prime, grad_out, o, aux, end, st, gp))) return rc;
    if (W > 1 && !ik && (rc = signal_peers(c, 3, n, st))) return rc;
  }
  if ((rc = finalize_step_outputs(c, s, st))) return rc;
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

// Bs[p]: rank p's batch; Rs[p] >= Bs[p]: its images (paired ones first, then its extra images); Ts[p] >= Bs[p]: its
// texts (paired ones first, then its hard negatives). Every argument is checked before the first CUDA call.
static int ctx_create_impl(siglip_ctx** out, int device, int rank, int world, const int* Bs, const int* Rs,
                           const int* Ts, int D, int DT = 0, int LM = 0) {
  if (out == nullptr) return fail(SIGLIP_ERR_INVALID, "out is null");
  *out = nullptr;
  if (world < 1 || world > kMaxWorld || rank < 0 || rank >= world)
    return fail(SIGLIP_ERR_INVALID, "rank/world out of range (world <= 32)");
  int Bmax = 0, Tmax = 0, Rmax = 0, Emax = 0;
  for (int p = 0; p < world; ++p) {
    if (Bs[p] < 1) return fail(SIGLIP_ERR_INVALID, "need B >= 1 on every rank");
    if (Ts[p] < Bs[p])
      return fail(SIGLIP_ERR_INVALID, "need texts_per_rank[p] >= batch_per_rank[p] (paired texts, then hard negatives)");
    if (Rs[p] < Bs[p])
      return fail(SIGLIP_ERR_INVALID, "need images_per_rank[p] >= batch_per_rank[p] (paired images, then extra images)");
    Bmax = Bs[p] > Bmax ? Bs[p] : Bmax;
    Tmax = Ts[p] > Tmax ? Ts[p] : Tmax;
    Rmax = Rs[p] > Rmax ? Rs[p] : Rmax;
    Emax = Rs[p] - Bs[p] > Emax ? Rs[p] - Bs[p] : Emax;
  }
  if (D < 8 || (D % 8) != 0) return fail(SIGLIP_ERR_INVALID, "need D a positive multiple of 8");
  if (DT < 0 || (DT % 8) != 0) return fail(SIGLIP_ERR_INVALID, "need D_teacher a positive multiple of 8 (0: no teacher)");
  if (LM < 0 || LM > SIGLIP_MAX_LABELS) return fail(SIGLIP_ERR_INVALID, "need 1 <= M <= SIGLIP_MAX_LABELS labels per set");
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
  for (int p = 0; p < world; ++p) {
    c->Bs[p] = Bs[p];
    c->Ts[p] = Ts[p];
    c->Rs[p] = Rs[p];
    c->extras = c->extras || Ts[p] != Bs[p];
    c->ximg = c->ximg || Rs[p] != Bs[p];
  }
  c->B = Bs[rank];
  c->T = Ts[rank];
  c->R = Rs[rank];
  c->Bmax = Bmax;
  c->Tmax = Tmax;
  c->Rmax = Rmax;
  c->Emax = Emax;
  c->own_pos_ids = c->R > c->B && c->T > c->B;
  c->D = D;
  c->DT = DT;
  c->LM = LM;
  c->Bp = round_up(Bmax, 256);
  c->Tp = round_up(Tmax, 256);
  c->Rp = round_up(Rmax, 256);
  for (int p = 0; p < world; ++p) {
    c->off[p + 1] = c->off[p] + Rs[p];
    c->toff[p + 1] = c->toff[p] + Ts[p];
  }
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
  CK(alloc(reinterpret_cast<void**>(&c->img16), static_cast<size_t>(c->R) * D * sizeof(__nv_bfloat16)));
  CK(alloc(reinterpret_cast<void**>(&c->partials), static_cast<size_t>(c->num_sms) * 4 * sizeof(double)));
  CK(alloc(reinterpret_cast<void**>(&c->fin_counter), sizeof(unsigned int)));
  CK(alloc(reinterpret_cast<void**>(&c->flags), kFlagBytes));
  CK(alloc(reinterpret_cast<void**>(&c->sync_words), kSyncWords * sizeof(unsigned int)));
  CK(alloc(reinterpret_cast<void**>(&c->scalars), 24 * sizeof(float)));
  // one slot per chunk holds its T ids (SIGLIP_OPT_EXTRA_TEXT_IDS may be set after the handle exchange, so the layout
  // cannot depend on it); without extras this is Bmax rounded up, as it was before they existed
  c->ids_stride = round_up(Tmax, 2);
  const size_t ids_slot_bytes = static_cast<size_t>(c->ids_stride) * sizeof(int64_t);
  if (LM > 0) {
    // a context with label sets holds its whole slot from the start (sets, text groups, then [R] image groups), and
    // its images' sets
    CK(alloc(reinterpret_cast<void**>(&c->ids_in), (ids_slot(c) + static_cast<size_t>(c->R)) * sizeof(int64_t)));
    c->ids_grp = true;
    CK(alloc(reinterpret_cast<void**>(&c->lrows), static_cast<size_t>(c->R) * LM * sizeof(int64_t)));
  } else {
    CK(alloc(reinterpret_cast<void**>(&c->ids_in), ids_slot_bytes));
  }
  if (c->R > c->B) CK(alloc(reinterpret_cast<void**>(&c->rids), static_cast<size_t>(c->R) * sizeof(int64_t)));
  if (c->own_pos_ids) {
    const int n = c->R > c->T ? c->R : c->T;
    std::vector<int64_t> iota(n);
    for (int i = 0; i < n; ++i) iota[i] = i;
    CK(alloc(reinterpret_cast<void**>(&c->iota), n * sizeof(int64_t)));
    CK(cudaMemcpy(c->iota, iota.data(), n * sizeof(int64_t), cudaMemcpyHostToDevice));
  }
  const size_t mkeys_bytes = 2 * mkeys_block(c) * sizeof(unsigned long long);
  c->w_stride = round_up(Tmax, 4);
  if (world > 1) {
    // the gathered ids, the two metric key blocks and the gathered text weights live behind the gathered text, so that
    // one exported handle covers all four (SIGLIP_OPT_SAMPLE_WEIGHTS may be set after the handle exchange, so the
    // weight slots exist whatever the options)
    const size_t w_bytes = static_cast<size_t>(world) * c->w_stride * sizeof(float);
    // a distillation context also gathers the teacher text there (nothing without a teacher)
    const size_t t_bytes = teacher_stride(c) * world * sizeof(__nv_bfloat16);
    // and the per-sample-loss partials behind that (sized whatever the options: a peer's offsets cannot depend on them)
    const size_t l_bytes = 2 * lsum_block(c) * sizeof(unsigned long long);
    // and the top-K column lists behind those (sized whatever the options, for the same reason)
    const size_t k_bytes = 2 * topk_cols_words(c) * sizeof(unsigned long long);
    // (every ids slot has a text-group half: SIGLIP_OPT_EXCLUDE_GROUPS may be set after the handle exchange too)
    CK(alloc(reinterpret_cast<void**>(&c->txt_all), stride * world * sizeof(__nv_bfloat16) + world * ids_slot(c) * 8 +
                                                        mkeys_bytes + w_bytes + t_bytes + l_bytes + k_bytes));
    c->ids_all = reinterpret_cast<int64_t*>(c->txt_all + stride * world);   // 16-byte aligned: D % 8 == 0
    c->mkeys[0] = reinterpret_cast<unsigned long long*>(reinterpret_cast<char*>(c->txt_all) + mkeys_offset(c));
    c->mkeys[1] = c->mkeys[0] + mkeys_block(c);
    c->w_all = reinterpret_cast<float*>(reinterpret_cast<char*>(c->txt_all) + weights_offset(c));
    if (DT > 0)
      c->ttxt_all = reinterpret_cast<__nv_bfloat16*>(reinterpret_cast<char*>(c->txt_all) + teacher_offset(c));
    c->lsum[0] = reinterpret_cast<unsigned long long*>(reinterpret_cast<char*>(c->txt_all) + lsum_offset(c));
    c->lsum[1] = c->lsum[0] + lsum_block(c);
    c->tk_cols[0] = reinterpret_cast<unsigned long long*>(reinterpret_cast<char*>(c->txt_all) + topk_offset(c));
    c->tk_cols[1] = c->tk_cols[0] + topk_cols_words(c);
    CK(alloc(reinterpret_cast<void**>(&c->slots), stride * world * sizeof(float)));
    CK(alloc(reinterpret_cast<void**>(&c->dimg_acc), static_cast<size_t>(c->R) * D * sizeof(float)));
    CK(alloc(reinterpret_cast<void**>(&c->dtxt_acc), static_cast<size_t>(c->T) * D * sizeof(float)));
    CK(alloc(reinterpret_cast<void**>(&c->reduce_ptrs_dev), world * sizeof(float*)));
    CK(alloc(reinterpret_cast<void**>(&c->final_ptrs_dev), 2 * sizeof(float*)));
    CK(alloc(reinterpret_cast<void**>(&c->signal_ptrs_dev), kFlagKinds * world * sizeof(unsigned int*)));
    CK(alloc(reinterpret_cast<void**>(&c->mailbox_ptrs_dev), world * sizeof(float*)));
    CK(alloc(reinterpret_cast<void**>(&c->mkey_ptrs_dev), 2 * world * sizeof(unsigned long long*)));
    CK(alloc(reinterpret_cast<void**>(&c->lsum_ptrs_dev), 2 * world * sizeof(unsigned long long*)));
    CK(alloc(reinterpret_cast<void**>(&c->tk_ptrs_dev), 2 * world * sizeof(unsigned long long*)));
    if (c->ximg) CK(alloc(reinterpret_cast<void**>(&c->xid_ptrs_dev), 2 * world * sizeof(int64_t*)));
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
  // The first sigma operand is allocated here when the device holds it. When the device is out of memory for it, the
  // context is created all the same and the first step allocates what it needs: a batch whose whole operand exceeds
  // the device runs under SIGLIP_OPT_SIGMA_BUDGET_MIB, and an unbounded step reports the shortfall there. Any other
  // failure fails the creation.
  {
    cudaError_t ge = cudaSuccess;
    if (int grc = ensure_g(c, 0, 0, &ge)) {
      if (ge != cudaErrorMemoryAllocation) return grc;
      g_last_error.clear();
    }
  }
  CK(cudaDeviceSynchronize());
  guard.c = nullptr;
  *out = c;
  return 0;
}

int siglip_ctx_create(siglip_ctx** out, int device, int rank, int world, int B, int D) {
  if (world < 1 || world > kMaxWorld) return fail(SIGLIP_ERR_INVALID, "rank/world out of range (world <= 32)");
  int Bs[kMaxWorld];
  for (int p = 0; p < world; ++p) Bs[p] = B;
  return ctx_create_impl(out, device, rank, world, Bs, Bs, Bs, D);
}

int siglip_ctx_create_uneven(siglip_ctx** out, int device, int rank, int world, const int* batch_per_rank, int D) {
  if (batch_per_rank == nullptr) return fail(SIGLIP_ERR_INVALID, "batch_per_rank is null");
  if (world < 1 || world > kMaxWorld) return fail(SIGLIP_ERR_INVALID, "rank/world out of range (world <= 32)");
  return ctx_create_impl(out, device, rank, world, batch_per_rank, batch_per_rank, batch_per_rank, D);
}

int siglip_ctx_create_texts(siglip_ctx** out, int device, int rank, int world, const int* images_per_rank,
                            const int* texts_per_rank, int D) {
  if (images_per_rank == nullptr || texts_per_rank == nullptr)
    return fail(SIGLIP_ERR_INVALID, "images_per_rank / texts_per_rank is null");
  if (world < 1 || world > kMaxWorld) return fail(SIGLIP_ERR_INVALID, "rank/world out of range (world <= 32)");
  return ctx_create_impl(out, device, rank, world, images_per_rank, images_per_rank, texts_per_rank, D);
}

int siglip_ctx_create_extras(siglip_ctx** out, int device, int rank, int world, const int* batch_per_rank,
                             const int* images_per_rank, const int* texts_per_rank, int D) {
  if (batch_per_rank == nullptr || images_per_rank == nullptr || texts_per_rank == nullptr)
    return fail(SIGLIP_ERR_INVALID, "batch_per_rank / images_per_rank / texts_per_rank is null");
  if (world < 1 || world > kMaxWorld) return fail(SIGLIP_ERR_INVALID, "rank/world out of range (world <= 32)");
  return ctx_create_impl(out, device, rank, world, batch_per_rank, images_per_rank, texts_per_rank, D);
}

// The public creation entries with a teacher or label sets: the lists are checked, then ctx_create_impl
static int ctx_create_checked(siglip_ctx** out, int device, int rank, int world, const int* Bs, const int* Rs,
                              const int* Ts, int D, int DT, int M, bool distill_opts = false) {
  if (Bs == nullptr || Rs == nullptr || Ts == nullptr)
    return fail(SIGLIP_ERR_INVALID, "batch_per_rank / images_per_rank / texts_per_rank is null");
  if (world < 1 || world > kMaxWorld) return fail(SIGLIP_ERR_INVALID, "rank/world out of range (world <= 32)");
  if (M < 0 || M > SIGLIP_MAX_LABELS)
    return fail(SIGLIP_ERR_INVALID, "need 1 <= M <= SIGLIP_MAX_LABELS labels per set (0: no label sets)");
  const int rc = ctx_create_impl(out, device, rank, world, Bs, Rs, Ts, D, DT, M);
  if (rc == 0) (*out)->distill_opts = distill_opts;
  return rc;
}

int siglip_ctx_create_distill(siglip_ctx** out, int device, int rank, int world, const int* batch_per_rank, int D,
                              int D_teacher) {
  if (batch_per_rank == nullptr) return fail(SIGLIP_ERR_INVALID, "batch_per_rank is null");
  return ctx_create_checked(out, device, rank, world, batch_per_rank, batch_per_rank, batch_per_rank, D, D_teacher, 0);
}

int siglip_ctx_create_labels(siglip_ctx** out, int device, int rank, int world, const int* batch_per_rank,
                             const int* images_per_rank, const int* texts_per_rank, int D, int M) {
  if (M < 1 || M > SIGLIP_MAX_LABELS) return fail(SIGLIP_ERR_INVALID, "need 1 <= M <= SIGLIP_MAX_LABELS labels per set");
  return ctx_create_checked(out, device, rank, world, batch_per_rank, images_per_rank, texts_per_rank, D, 0, M);
}

int siglip_ctx_create_distill_extras(siglip_ctx** out, int device, int rank, int world, const int* batch_per_rank,
                                     const int* images_per_rank, const int* texts_per_rank, int D, int D_teacher,
                                     int M) {
  if (D_teacher < 8) return fail(SIGLIP_ERR_INVALID, "need D_teacher a positive multiple of 8");
  return ctx_create_checked(out, device, rank, world, batch_per_rank, images_per_rank, texts_per_rank, D, D_teacher, M,
                            true);
}

int siglip_set_teacher(siglip_ctx* c, const void* timg, const void* ttxt, int teacher_f16, const float* t_prime_T,
                       const float* bias_T, float lambda) {
  if (c == nullptr || timg == nullptr || ttxt == nullptr || t_prime_T == nullptr || bias_T == nullptr)
    return fail(SIGLIP_ERR_INVALID, "null argument");
  if (!c->distill) return fail(SIGLIP_ERR_STATE, "siglip_set_teacher needs SIGLIP_OPT_DISTILL = 1");
  if (!(lambda > 0.0f && lambda <= 1.0f)) return fail(SIGLIP_ERR_INVALID, "distillation lambda must be in (0, 1]");
  if (teacher_f16 != 0 && teacher_f16 != 1) return fail(SIGLIP_ERR_INVALID, "teacher_f16 must be 0 or 1");
  if ((reinterpret_cast<uintptr_t>(timg) | reinterpret_cast<uintptr_t>(ttxt)) & 15u)
    return fail(SIGLIP_ERR_INVALID, "teacher embeddings must be 16-byte aligned");
  c->t_img = timg;
  c->t_txt = ttxt;
  c->t_f16 = teacher_f16;
  c->t_tprime = t_prime_T;
  c->t_bias = bias_T;
  c->t_lambda = lambda;
  c->teacher_set = true;
  return 0;
}

int siglip_ctx_set_option(siglip_ctx* c, int option, int value) {
  if (c == nullptr) return fail(SIGLIP_ERR_INVALID, "ctx is null");
  switch (option) {
    case SIGLIP_OPT_DISTILL:
      if (value && c->DT == 0)
        return fail(SIGLIP_ERR_STATE,
                    "SIGLIP_OPT_DISTILL needs a context created with siglip_ctx_create_distill(_extras)");
      if (value && c->exclude_groups && !c->distill_opts)
        return fail(SIGLIP_ERR_STATE, "SIGLIP_OPT_DISTILL is unavailable under SIGLIP_OPT_EXCLUDE_GROUPS on a "
                                      "siglip_ctx_create_distill context (siglip_ctx_create_distill_extras takes both)");
      if (value && c->focal)
        return fail(SIGLIP_ERR_STATE, "SIGLIP_OPT_DISTILL is unavailable under SIGLIP_OPT_FOCAL");
      c->distill = value ? 1 : 0;
      c->teacher_set = false;
      return 0;
    case SIGLIP_OPT_EXCLUDE_GROUPS: {
      if (value && c->distill && !c->distill_opts)
        return fail(SIGLIP_ERR_STATE, "SIGLIP_OPT_EXCLUDE_GROUPS is unavailable under SIGLIP_OPT_DISTILL on a "
                                      "siglip_ctx_create_distill context (siglip_ctx_create_distill_extras takes both)");
      if (value && !c->ids_grp) {
        // ids_in grows its group halves ([ids_stride] text groups, [R] image groups) on first use, so a context that
        // never turns the mode on holds the workspace it held without it. Its ids are kept (they may be set already).
        CK(cudaSetDevice(c->device));
        CK(cudaDeviceSynchronize());   // no launch in flight reads the old buffer
        const size_t bytes = (ids_slot(c) + static_cast<size_t>(c->R)) * sizeof(int64_t);
        int64_t* buf = nullptr;
        CK(cudaMalloc(reinterpret_cast<void**>(&buf), bytes));
        CK(cudaMemset(buf, 0, bytes));
        CK(cudaMemcpy(buf, c->ids_in, static_cast<size_t>(c->ids_stride) * sizeof(int64_t), cudaMemcpyDeviceToDevice));
        CK(cudaFree(c->ids_in));
        c->ids_in = buf;
        c->ids_grp = true;
        c->workspace_bytes += bytes - static_cast<size_t>(c->ids_stride) * sizeof(int64_t);
      }
      c->exclude_groups = value ? 1 : 0;
      c->groups_set = false;
      return 0;
    }
    case SIGLIP_OPT_LABEL_SETS:
      if (value && c->LM == 0)
        return fail(SIGLIP_ERR_STATE,
                    "SIGLIP_OPT_LABEL_SETS needs a context created with siglip_ctx_create_labels or with M > 0");
      if (value && (c->sample_ids || c->extra_text_ids || c->extra_image_ids))
        return fail(SIGLIP_ERR_STATE, "SIGLIP_OPT_LABEL_SETS replaces sample ids: turn SIGLIP_OPT_SAMPLE_IDS off first");
      c->label_sets = value ? 1 : 0;
      c->sets_set = false;
      return 0;
    case SIGLIP_OPT_FOCAL:
      if (value && c->distill)
        return fail(SIGLIP_ERR_STATE, "SIGLIP_OPT_FOCAL is unavailable under SIGLIP_OPT_DISTILL");
      c->focal = value ? 1 : 0;
      return 0;
    case SIGLIP_OPT_SIGMA_BUDGET_MIB:
      if (value < 0) return fail(SIGLIP_ERR_INVALID, "the sigma budget must be >= 0 MiB (0: unbounded)");
      c->sigma_budget_mib = value;
      // the operands are allocated again, at the height the next step needs
      CK(cudaSetDevice(c->device));
      for (int i = 0; i < kMaxWorld; ++i) release_g(c, i);
      c->gen = 0;
      return 0;
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
    case SIGLIP_OPT_GRAD_TILE_N:
      if (value != 0 && value != 128 && value != 256) return fail(SIGLIP_ERR_INVALID, "grad_tile_n must be 0, 128 or 256");
      c->grad_tile_n = value;
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
    case SIGLIP_OPT_SAMPLE_IDS:
      if (value && c->label_sets)
        return fail(SIGLIP_ERR_STATE, "SIGLIP_OPT_SAMPLE_IDS is unavailable under SIGLIP_OPT_LABEL_SETS");
      c->sample_ids = value ? 1 : 0;
      c->ids_set = false;
      if (!c->sample_ids) c->extra_text_ids = c->extra_image_ids = 0;   // the extras' ids extend the sample ids
      c->extra_ids_set = false;
      c->ximg_ids_set = false;
      return 0;
    case SIGLIP_OPT_EXTRA_IMAGE_IDS:
      if (value && c->label_sets)
        return fail(SIGLIP_ERR_STATE, "SIGLIP_OPT_EXTRA_IMAGE_IDS is unavailable under SIGLIP_OPT_LABEL_SETS");
      if (value && !c->sample_ids)
        return fail(SIGLIP_ERR_STATE, "SIGLIP_OPT_EXTRA_IMAGE_IDS needs SIGLIP_OPT_SAMPLE_IDS on first");
      c->extra_image_ids = value ? 1 : 0;
      c->ximg_ids_set = false;
      return 0;
    case SIGLIP_OPT_EXTRA_TEXT_IDS:
      if (value && c->label_sets)
        return fail(SIGLIP_ERR_STATE, "SIGLIP_OPT_EXTRA_TEXT_IDS is unavailable under SIGLIP_OPT_LABEL_SETS");
      if (value && !c->sample_ids)
        return fail(SIGLIP_ERR_STATE, "SIGLIP_OPT_EXTRA_TEXT_IDS needs SIGLIP_OPT_SAMPLE_IDS on first");
      c->extra_text_ids = value ? 1 : 0;
      c->extra_ids_set = false;
      return 0;
    case SIGLIP_OPT_SAMPLE_WEIGHTS:
      c->sample_weights = value ? 1 : 0;
      c->weights_set = false;
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

int siglip_ctx_sigma_panels(const siglip_ctx* c, int buffers, int* panel_rows, int* panels, int* whole) {
  if (c == nullptr || buffers < 0 || buffers > kMaxWorld) return fail(SIGLIP_ERR_INVALID, "invalid argument");
  const Panels pn = sigma_panels(c->R, c->Rp, c->Tp, buffers ? buffers : fused_buffers(c), panel_unit(c),
                                 c->sigma_budget_mib);
  if (panel_rows != nullptr) *panel_rows = pn.rows;
  if (panels != nullptr) *panels = pn.rows ? pn.n : 0;
  if (whole != nullptr) *whole = (pn.rows == c->R && pn.buf_rows == c->Rp) ? 1 : 0;
  return 0;
}

int siglip_sigma_panel_rows(int rows, int rows_padded, int cols_padded, int buffers, int cluster_rows, int budget_mib,
                            int* buffer_rows) {
  if (rows < 1 || rows_padded < rows || cols_padded < 1 || buffers < 1 || cluster_rows < 1 || budget_mib < 0)
    return -fail(SIGLIP_ERR_INVALID, "siglip_sigma_panel_rows: invalid argument");
  const Panels pn = sigma_panels(rows, rows_padded, cols_padded, buffers, cluster_rows, budget_mib);
  if (buffer_rows != nullptr) *buffer_rows = pn.buf_rows;
  return pn.rows;
}

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
  b.T = c->T;
  b.Tmax = c->Tmax;
  b.R = c->R;
  b.Rmax = c->Rmax;
  b.D_teacher = c->DT;
  b.M = c->LM;
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
  // every rank's column partial of my chunk, per step parity (loopback: the stand-ins siglip_debug_set_peer_metric_keys
  // seeds)
  std::vector<const unsigned long long*> mk(2 * c->world);
  for (int q = 0; q < 2; ++q)
    for (int p = 0; p < c->world; ++p) {
      const unsigned long long* blk =
          reinterpret_cast<const unsigned long long*>(reinterpret_cast<const char*>(c->peer_txt[p]) + mkeys_offset(c)) +
          q * mkeys_block(c);
      mk[q * c->world + p] = blk + static_cast<size_t>(c->rank) * c->Tmax;
      if (c->loopback && p != c->rank) mk[q * c->world + p] = c->loop_keys + static_cast<size_t>(p) * c->Tmax;
    }
  CK(cudaMemcpy(c->mkey_ptrs_dev, mk.data(), mk.size() * sizeof(unsigned long long*), cudaMemcpyHostToDevice));
  // every rank's loss column partial of my chunk, per step parity (loopback: the stand-ins
  // siglip_debug_set_peer_sample_loss_partials seeds, with their poison words at the same distance)
  std::vector<const unsigned long long*> ls(2 * c->world);
  for (int q = 0; q < 2; ++q)
    for (int p = 0; p < c->world; ++p) {
      const unsigned long long* blk =
          reinterpret_cast<const unsigned long long*>(reinterpret_cast<const char*>(c->peer_txt[p]) + lsum_offset(c)) +
          q * lsum_block(c);
      if (c->loopback && p != c->rank) blk = c->loop_lsums + static_cast<size_t>(p) * lsum_block(c);
      ls[q * c->world + p] = blk + static_cast<size_t>(c->rank) * c->Tmax;
    }
  CK(cudaMemcpy(c->lsum_ptrs_dev, ls.data(), ls.size() * sizeof(unsigned long long*), cudaMemcpyHostToDevice));
  // every rank's top-K column lists of my chunk, per step parity (loopback: the stand-ins
  // siglip_debug_set_peer_topk_keys seeds)
  std::vector<const unsigned long long*> tk(2 * c->world);
  for (int q = 0; q < 2; ++q)
    for (int p = 0; p < c->world; ++p) {
      const unsigned long long* blk =
          reinterpret_cast<const unsigned long long*>(reinterpret_cast<const char*>(c->peer_txt[p]) + topk_offset(c)) +
          q * topk_cols_words(c) + static_cast<size_t>(c->rank) * c->Tmax * siglip::kTopKMax;
      if (c->loopback && p != c->rank) blk = c->loop_topk + static_cast<size_t>(p) * c->Tmax * siglip::kTopKMax;
      tk[q * c->world + p] = blk;
    }
  CK(cudaMemcpy(c->tk_ptrs_dev, tk.data(), tk.size() * sizeof(unsigned long long*), cudaMemcpyHostToDevice));
  if (c->xid_ptrs_dev != nullptr) {
    // every rank's published extra-image ids, per step parity (loopback: the stand-ins
    // siglip_debug_set_peer_extra_image_ids seeds)
    std::vector<const int64_t*> xi(2 * c->world);
    for (int q = 0; q < 2; ++q)
      for (int p = 0; p < c->world; ++p) {
        xi[q * c->world + p] = reinterpret_cast<const int64_t*>(
            reinterpret_cast<const unsigned long long*>(reinterpret_cast<const char*>(c->peer_txt[p]) + mkeys_offset(c)) +
            q * mkeys_block(c) + mkeys_xids(c));
        if (c->loopback && p != c->rank)
          xi[q * c->world + p] = c->loop_xids + static_cast<size_t>(p) * loop_xids_stride(c);
      }
    CK(cudaMemcpy(c->xid_ptrs_dev, xi.data(), xi.size() * sizeof(int64_t*), cudaMemcpyHostToDevice));
  }
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
    if (b.T != c->Ts[p] || b.Tmax != c->Tmax)
      return fail(SIGLIP_ERR_INVALID,
                  "peer context has a different text count than this rank was told: every rank must be created with the "
                  "same texts_per_rank list (siglip_ctx_create_texts; batch + hard negatives per rank)");
    if (b.R != c->Rs[p] || b.Rmax != c->Rmax)
      return fail(SIGLIP_ERR_INVALID,
                  "peer context has a different image count than this rank was told: every rank must be created with "
                  "the same images_per_rank list (siglip_ctx_create_extras; batch + extra images per rank)");
    if (b.D_teacher != c->DT)
      return fail(SIGLIP_ERR_INVALID,
                  "peer context has a different D_teacher than this rank: every rank must be created with the same "
                  "siglip_ctx_create_distill arguments");
    if (b.M != c->LM)
      return fail(SIGLIP_ERR_INVALID,
                  "peer context has a different label-set width M than this rank: every rank must be created with the "
                  "same siglip_ctx_create_labels M");
    if (p == c->rank) continue;
    char me[sizeof(b.host)] = {0};
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

int siglip_set_sample_ids(siglip_ctx* c, const int64_t* ids_dev, void* cuda_stream) {
  if (c == nullptr || ids_dev == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (!c->sample_ids) return fail(SIGLIP_ERR_STATE, "siglip_set_sample_ids needs SIGLIP_OPT_SAMPLE_IDS = 1");
  CK(cudaSetDevice(c->device));
  CK(cudaMemcpyAsync(c->ids_in, ids_dev, ids_bytes(c, c->rank), cudaMemcpyDeviceToDevice,
                     static_cast<cudaStream_t>(cuda_stream)));
  if (c->rids != nullptr)   // the paired images' ids head my row ids too
    CK(cudaMemcpyAsync(c->rids, ids_dev, ids_bytes(c, c->rank), cudaMemcpyDeviceToDevice,
                       static_cast<cudaStream_t>(cuda_stream)));
  c->ids_set = true;
  return 0;
}

int siglip_set_extra_image_ids(siglip_ctx* c, const int64_t* ids_dev, void* cuda_stream) {
  if (c == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  // behind this rank's B sample ids in its private row ids: the [R] ids of my images
  const size_t e = static_cast<size_t>(c->R - c->B);
  if (ids_dev == nullptr && e > 0) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (!c->extra_image_ids)
    return fail(SIGLIP_ERR_STATE, "siglip_set_extra_image_ids needs SIGLIP_OPT_EXTRA_IMAGE_IDS on");
  CK(cudaSetDevice(c->device));
  if (e > 0)
    CK(cudaMemcpyAsync(c->rids + c->B, ids_dev, e * sizeof(int64_t), cudaMemcpyDeviceToDevice,
                       static_cast<cudaStream_t>(cuda_stream)));
  c->ximg_ids_set = true;
  return 0;
}

int siglip_set_extra_text_ids(siglip_ctx* c, const int64_t* ids_dev, void* cuda_stream) {
  if (c == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  // behind this rank's B sample ids: ids_in is then the [T] id list of my text chunk
  const size_t k = static_cast<size_t>(c->T - c->B);
  if (ids_dev == nullptr && k > 0) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (!c->extra_text_ids)
    return fail(SIGLIP_ERR_STATE, "siglip_set_extra_text_ids needs SIGLIP_OPT_EXTRA_TEXT_IDS on");
  CK(cudaSetDevice(c->device));
  if (k > 0)
    CK(cudaMemcpyAsync(c->ids_in + c->B, ids_dev, k * sizeof(int64_t), cudaMemcpyDeviceToDevice,
                       static_cast<cudaStream_t>(cuda_stream)));
  c->extra_ids_set = true;
  return 0;
}

// the weight buffer of my chunk and images, allocated on the first call like the metric keys (so a context that never
// uses weights holds the workspace it held without them; allowed inside a CUDA-graph capture)
static int ensure_weights(siglip_ctx* c) {
  if (c->w_in != nullptr) return 0;
  const size_t bytes = (static_cast<size_t>(c->w_stride) + c->R) * sizeof(float);
  cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
  CK(cudaThreadExchangeStreamCaptureMode(&mode));
  float* w = nullptr;
  const cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&w), bytes);
  cudaThreadExchangeStreamCaptureMode(&mode);
  CK(e);
  c->w_in = w;
  c->workspace_bytes += bytes;
  return 0;
}

int siglip_set_sample_weights(siglip_ctx* c, const float* image_w, const float* text_w, void* cuda_stream) {
  if (c == nullptr) return fail(SIGLIP_ERR_INVALID, "ctx is null");
  if (!c->sample_weights)
    return fail(SIGLIP_ERR_STATE, "siglip_set_sample_weights needs SIGLIP_OPT_SAMPLE_WEIGHTS = 1");
  CK(cudaSetDevice(c->device));
  int rc;
  if ((rc = ensure_weights(c))) return rc;
  CKI(siglip::launch_clamp_weights(text_w, c->w_in, c->T, image_w, c->w_in + c->w_stride, c->R,
                                   static_cast<cudaStream_t>(cuda_stream)));
  c->launches++;
  c->weights_set = true;
  return 0;
}

int siglip_set_groups(siglip_ctx* c, const int64_t* image_groups, const int64_t* text_groups, void* cuda_stream) {
  if (c == nullptr || image_groups == nullptr || text_groups == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (!c->exclude_groups) return fail(SIGLIP_ERR_STATE, "siglip_set_groups needs SIGLIP_OPT_EXCLUDE_GROUPS = 1");
  CK(cudaSetDevice(c->device));
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  // my text groups go to the group half of my slot (published with my ids), my image groups behind it
  CK(cudaMemcpyAsync(c->ids_in + set_words(c), text_groups, static_cast<size_t>(c->T) * sizeof(int64_t),
                     cudaMemcpyDeviceToDevice, st));
  CK(cudaMemcpyAsync(c->ids_in + ids_slot(c), image_groups, static_cast<size_t>(c->R) * sizeof(int64_t),
                     cudaMemcpyDeviceToDevice, st));
  c->groups_set = true;
  return 0;
}

int siglip_set_label_sets(siglip_ctx* c, const int64_t* sample_labels, const int64_t* extra_text_labels,
                          const int64_t* extra_image_labels, void* cuda_stream) {
  if (c == nullptr || sample_labels == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (!c->label_sets) return fail(SIGLIP_ERR_STATE, "siglip_set_label_sets needs SIGLIP_OPT_LABEL_SETS = 1");
  CK(cudaSetDevice(c->device));
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  const size_t m = static_cast<size_t>(c->LM), w = sizeof(int64_t);
  // a sample's set belongs to its image (my rows) and to its paired text (the set half of my slot, published)
  CK(cudaMemcpyAsync(c->lrows, sample_labels, c->B * m * w, cudaMemcpyDeviceToDevice, st));
  CK(cudaMemcpyAsync(c->ids_in, sample_labels, c->B * m * w, cudaMemcpyDeviceToDevice, st));
  // extras without sets (null) get empty ones: all bytes 0xff is -1 in every slot
  if (c->T > c->B) {
    if (extra_text_labels != nullptr)
      CK(cudaMemcpyAsync(c->ids_in + c->B * m, extra_text_labels, (c->T - c->B) * m * w, cudaMemcpyDeviceToDevice, st));
    else
      CK(cudaMemsetAsync(c->ids_in + c->B * m, 0xff, (c->T - c->B) * m * w, st));
  }
  if (c->R > c->B) {
    if (extra_image_labels != nullptr)
      CK(cudaMemcpyAsync(c->lrows + c->B * m, extra_image_labels, (c->R - c->B) * m * w, cudaMemcpyDeviceToDevice, st));
    else
      CK(cudaMemsetAsync(c->lrows + c->B * m, 0xff, (c->R - c->B) * m * w, st));
  }
  c->sets_set = true;
  return 0;
}

int siglip_set_focal(siglip_ctx* c, float gamma, float alpha) {
  if (c == nullptr) return fail(SIGLIP_ERR_INVALID, "ctx is null");
  if (!c->focal) return fail(SIGLIP_ERR_STATE, "siglip_set_focal needs SIGLIP_OPT_FOCAL = 1");
  // |g| < 1.44 for gamma <= 8, so g * kGScale stays inside the fp16 sigma operand (DESIGN.md, "Focal pair loss")
  if (!(gamma >= 0.0f && gamma <= 8.0f)) return fail(SIGLIP_ERR_INVALID, "focal gamma must be finite and in [0, 8]");
  if (alpha != alpha || alpha > 1.0f) return fail(SIGLIP_ERR_INVALID, "focal alpha must be in [0, 1], or < 0 for none");
  c->focal_gamma = gamma;
  c->focal_alpha = alpha < 0.0f ? -1.0f : alpha;
  c->focal_set = true;
  return 0;
}

// one rank: the key blocks are allocated on the first request that reduces argmax keys (siglip_request_metrics, or
// siglip_request_topk with K = 1), so a context that never asks holds exactly the workspace it held without them.
// (world > 1: they are part of the exported text allocation.) The allocation is not a stream operation; the relaxed
// capture mode lets a first request inside a CUDA-graph capture make it, as PyTorch's caching allocator does.
static int ensure_metric_keys(siglip_ctx* c) {
  if (c->mkeys[0] != nullptr) return 0;
  const size_t bytes = 2 * mkeys_block(c) * sizeof(unsigned long long);
  CK(cudaSetDevice(c->device));
  cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
  CK(cudaThreadExchangeStreamCaptureMode(&mode));
  unsigned long long* keys = nullptr;
  const cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&keys), bytes);
  cudaThreadExchangeStreamCaptureMode(&mode);
  CK(e);
  c->mkeys[0] = keys;
  c->mkeys[1] = keys + mkeys_block(c);
  c->workspace_bytes += bytes;
  return 0;
}

int siglip_request_metrics(siglip_ctx* c, float* top1, int64_t* i2t_index, int64_t* t2i_index) {
  if (c == nullptr || top1 == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument (top1 is required)");
  int rc;
  if ((rc = ensure_metric_keys(c))) return rc;
  c->m_top1 = top1;
  c->m_i2t = i2t_index;
  c->m_t2i = t2i_index;
  c->metrics_armed = true;
  return 0;
}

int siglip_request_sample_losses(siglip_ctx* c, float* image_loss, float* text_loss) {
  if (c == nullptr || image_loss == nullptr || text_loss == nullptr)
    return fail(SIGLIP_ERR_INVALID, "null argument (image_loss and text_loss are required)");
  if (c->distill && !c->distill_opts)
    return fail(SIGLIP_ERR_STATE, "per-sample losses are unavailable under SIGLIP_OPT_DISTILL on a "
                                  "siglip_ctx_create_distill context (siglip_ctx_create_distill_extras takes them)");
  if (c->lsum[0] == nullptr) {
    // one rank: the blocks are allocated on the first request, as the metric keys are (and apart from them), so a
    // context that never asks holds exactly the workspace it held without them; allowed inside a CUDA-graph capture
    const size_t bytes = 2 * lsum_block(c) * sizeof(unsigned long long);
    CK(cudaSetDevice(c->device));
    cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
    CK(cudaThreadExchangeStreamCaptureMode(&mode));
    unsigned long long* words = nullptr;
    const cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&words), bytes);
    cudaThreadExchangeStreamCaptureMode(&mode);
    CK(e);
    c->lsum[0] = words;
    c->lsum[1] = words + lsum_block(c);
    c->workspace_bytes += bytes;
  }
  c->l_img = image_loss;
  c->l_txt = text_loss;
  c->losses_armed = true;
  return 0;
}

int siglip_request_topk(siglip_ctx* c, int k, float* recall, int64_t* i2t_topk, int64_t* t2i_topk) {
  if (c == nullptr || recall == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument (recall is required)");
  if (k < 1 || k > SIGLIP_TOPK_MAX) return fail(SIGLIP_ERR_INVALID, "k must be in 1 .. SIGLIP_TOPK_MAX");
  if (c->distill && !c->distill_opts)
    return fail(SIGLIP_ERR_STATE, "top-K retrieval is unavailable under SIGLIP_OPT_DISTILL on a "
                                  "siglip_ctx_create_distill context (siglip_ctx_create_distill_extras takes it)");
  int rc;
  if (k == 1 && (rc = ensure_metric_keys(c))) return rc;   // K = 1 runs the metrics path on the argmax keys
  if (k > 1 && c->tk_rows[0] == nullptr) {
    // the row lists (and on one rank the column lists ahead of them) are allocated by the first request, so a context
    // that never asks holds exactly the workspace it held without them; allowed inside a CUDA-graph capture
    const size_t cols = (c->world == 1) ? 2 * topk_cols_words(c) : 0;
    const size_t bytes = (cols + 2 * topk_rows_words(c)) * sizeof(unsigned long long);
    CK(cudaSetDevice(c->device));
    cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
    CK(cudaThreadExchangeStreamCaptureMode(&mode));
    unsigned long long* words = nullptr;
    const cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&words), bytes);
    cudaThreadExchangeStreamCaptureMode(&mode);
    CK(e);
    if (c->world == 1) {
      c->tk_cols[0] = words + 2 * topk_rows_words(c);   // behind the row lists, which free_ctx releases
      c->tk_cols[1] = c->tk_cols[0] + topk_cols_words(c);
    }
    c->tk_rows[0] = words;
    c->tk_rows[1] = words + topk_rows_words(c);
    c->workspace_bytes += bytes;
  }
  c->topk_k = k;
  c->k_recall = recall;
  c->k_i2t = i2t_topk;
  c->k_t2i = t2i_topk;
  c->topk_armed = true;
  return 0;
}

int siglip_debug_set_peer_topk_keys(siglip_ctx* c, int peer, const uint64_t* keys_dev, void* cuda_stream) {
  if (c == nullptr || keys_dev == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (!c->loopback || peer < 0 || peer >= c->world || peer == c->rank)
    return fail(SIGLIP_ERR_INVALID, "siglip_debug_set_peer_topk_keys needs a loopback context and a peer rank != own rank");
  CK(cudaSetDevice(c->device));
  CK(cudaMemcpyAsync(c->loop_topk + static_cast<size_t>(peer) * c->Tmax * siglip::kTopKMax, keys_dev,
                     static_cast<size_t>(c->T) * siglip::kTopKMax * sizeof(uint64_t), cudaMemcpyDeviceToDevice,
                     static_cast<cudaStream_t>(cuda_stream)));
  return 0;
}

int siglip_debug_set_peer_sample_loss_partials(siglip_ctx* c, int peer, const int64_t* partials_dev,
                                               void* cuda_stream) {
  if (c == nullptr || partials_dev == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (!c->loopback || peer < 0 || peer >= c->world || peer == c->rank)
    return fail(SIGLIP_ERR_INVALID,
                "siglip_debug_set_peer_sample_loss_partials needs a loopback context and a peer rank != own rank");
  CK(cudaSetDevice(c->device));
  CK(cudaMemcpyAsync(c->loop_lsums + static_cast<size_t>(peer) * lsum_block(c) + static_cast<size_t>(c->rank) * c->Tmax,
                     partials_dev, static_cast<size_t>(c->T) * sizeof(int64_t), cudaMemcpyDeviceToDevice,
                     static_cast<cudaStream_t>(cuda_stream)));
  return 0;
}

int siglip_debug_set_peer_sample_loss_poison(siglip_ctx* c, int peer, const int64_t* poison_dev, void* cuda_stream) {
  if (c == nullptr || poison_dev == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (!c->loopback || peer < 0 || peer >= c->world || peer == c->rank)
    return fail(SIGLIP_ERR_INVALID,
                "siglip_debug_set_peer_sample_loss_poison needs a loopback context and a peer rank != own rank");
  CK(cudaSetDevice(c->device));
  // the poison words sit lsum_half words behind the sums siglip_debug_set_peer_sample_loss_partials seeds
  CK(cudaMemcpyAsync(c->loop_lsums + static_cast<size_t>(peer) * lsum_block(c) + lsum_half(c) +
                         static_cast<size_t>(c->rank) * c->Tmax,
                     poison_dev, static_cast<size_t>(c->T) * sizeof(int64_t), cudaMemcpyDeviceToDevice,
                     static_cast<cudaStream_t>(cuda_stream)));
  return 0;
}

int siglip_debug_set_peer_metric_keys(siglip_ctx* c, int peer, const uint64_t* keys_dev, void* cuda_stream) {
  if (c == nullptr || keys_dev == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (!c->loopback || peer < 0 || peer >= c->world || peer == c->rank)
    return fail(SIGLIP_ERR_INVALID,
                "siglip_debug_set_peer_metric_keys needs a loopback context and a peer rank != own rank");
  CK(cudaSetDevice(c->device));
  // the keys of the texts the finalisation ranks: all T under label sets (their t2i ranks every text)
  const int n = c->label_sets ? c->T : chunk_id_count(c, c->rank);
  CK(cudaMemcpyAsync(c->loop_keys + static_cast<size_t>(peer) * c->Tmax, keys_dev,
                     static_cast<size_t>(n) * sizeof(unsigned long long),
                     cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(cuda_stream)));
  return 0;
}

int siglip_debug_set_peer_extra_image_ids(siglip_ctx* c, int peer, const int64_t* ids_dev, void* cuda_stream) {
  if (c == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (!c->loopback || peer < 0 || peer >= c->world || peer == c->rank)
    return fail(SIGLIP_ERR_INVALID,
                "siglip_debug_set_peer_extra_image_ids needs a loopback context and a peer rank != own rank");
  const size_t e = static_cast<size_t>(c->Rs[peer] - c->Bs[peer]);
  if (e == 0) return 0;
  if (ids_dev == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  CK(cudaSetDevice(c->device));
  CK(cudaMemcpyAsync(c->loop_xids + static_cast<size_t>(peer) * loop_xids_stride(c), ids_dev, e * sizeof(int64_t),
                     cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(cuda_stream)));
  return 0;
}

int siglip_debug_set_peer_extra_image_label_sets(siglip_ctx* c, int peer, const int64_t* sets_dev, void* cuda_stream) {
  if (c == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (!c->loopback || peer < 0 || peer >= c->world || peer == c->rank || c->LM == 0)
    return fail(SIGLIP_ERR_INVALID,
                "siglip_debug_set_peer_extra_image_label_sets needs a loopback labels context and a peer rank != own "
                "rank");
  const size_t e = static_cast<size_t>(c->Rs[peer] - c->Bs[peer]) * c->LM;
  if (e == 0) return 0;
  if (sets_dev == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  CK(cudaSetDevice(c->device));
  CK(cudaMemcpyAsync(c->loop_xids + static_cast<size_t>(peer) * loop_xids_stride(c), sets_dev, e * sizeof(int64_t),
                     cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(cuda_stream)));
  return 0;
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
  if (c->sample_ids)
    return fail(SIGLIP_ERR_STATE, "the host-buffer entries take no sample ids: unavailable under SIGLIP_OPT_SAMPLE_IDS");
  if (c->extras)
    return fail(SIGLIP_ERR_STATE,
                "the host-buffer entries stage [B, D] text: unavailable for a context with hard negatives "
                "(siglip_ctx_create_texts with texts_per_rank != images_per_rank)");
  if (c->ximg)
    return fail(SIGLIP_ERR_STATE,
                "the host-buffer entries stage [B, D] images: unavailable for a context with extra images "
                "(siglip_ctx_create_extras with images_per_rank != batch_per_rank)");
  if (c->metrics_armed)
    return fail(SIGLIP_ERR_STATE, "the host-buffer entries return no retrieval metrics: siglip_request_metrics is armed");
  if (c->losses_armed)
    return fail(SIGLIP_ERR_STATE,
                "the host-buffer entries return no per-sample losses: siglip_request_sample_losses is armed");
  if (c->topk_armed)
    return fail(SIGLIP_ERR_STATE, "the host-buffer entries return no top-K lists: siglip_request_topk is armed");
  if (c->sample_weights)
    return fail(SIGLIP_ERR_STATE,
                "the host-buffer entries take no sample weights: unavailable under SIGLIP_OPT_SAMPLE_WEIGHTS");
  if (c->distill)
    return fail(SIGLIP_ERR_STATE, "the host-buffer entries take no teacher: unavailable under SIGLIP_OPT_DISTILL");
  if (c->exclude_groups)
    return fail(SIGLIP_ERR_STATE,
                "the host-buffer entries take no group ids: unavailable under SIGLIP_OPT_EXCLUDE_GROUPS");
  if (c->label_sets)
    return fail(SIGLIP_ERR_STATE,
                "the host-buffer entries take no label sets: unavailable under SIGLIP_OPT_LABEL_SETS");
  if (c->focal)
    return fail(SIGLIP_ERR_STATE, "the host-buffer entries compute the SigLIP loss: unavailable under SIGLIP_OPT_FOCAL");
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
    CK(cudaMalloc(reinterpret_cast<void**>(&c->loop_keys), static_cast<size_t>(c->world) * c->Tmax * 8));
    CK(cudaMemset(c->loop_keys, 0, static_cast<size_t>(c->world) * c->Tmax * 8));
    CK(cudaMalloc(reinterpret_cast<void**>(&c->loop_lsums), static_cast<size_t>(c->world) * lsum_block(c) * 8));
    CK(cudaMemset(c->loop_lsums, 0, static_cast<size_t>(c->world) * lsum_block(c) * 8));
    CK(cudaMalloc(reinterpret_cast<void**>(&c->loop_topk), topk_cols_words(c) * 8));
    CK(cudaMemset(c->loop_topk, 0, topk_cols_words(c) * 8));
    if (c->Emax > 0) {
      CK(cudaMalloc(reinterpret_cast<void**>(&c->loop_xids), static_cast<size_t>(c->world) * loop_xids_stride(c) * 8));
      CK(cudaMemset(c->loop_xids, 0, static_cast<size_t>(c->world) * loop_xids_stride(c) * 8));
    }
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
                     static_cast<size_t>(c->Ts[chunk]) * c->D * sizeof(__nv_bfloat16), cudaMemcpyDeviceToDevice,
                     static_cast<cudaStream_t>(cuda_stream)));
  return 0;
}

int siglip_debug_set_teacher_text_chunk(siglip_ctx* c, int chunk, const void* ttxt_dev, void* cuda_stream) {
  if (c == nullptr || ttxt_dev == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (c->DT == 0) return fail(SIGLIP_ERR_STATE, "not a distillation context (siglip_ctx_create_distill)");
  if (c->world == 1 || chunk < 0 || chunk >= c->world) return fail(SIGLIP_ERR_INVALID, "chunk out of range");
  CK(cudaMemcpyAsync(c->ttxt_all + chunk * teacher_stride(c), ttxt_dev, teacher_chunk_bytes(c, chunk),
                     cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(cuda_stream)));
  return 0;
}

int siglip_teacher_convert_f32(siglip_ctx* c, int rows, const float* x_f32, void* out_16bit, int f16,
                               void* cuda_stream) {
  if (c == nullptr || x_f32 == nullptr || out_16bit == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (c->DT == 0) return fail(SIGLIP_ERR_STATE, "not a distillation context (siglip_ctx_create_distill)");
  if (rows < 1) return fail(SIGLIP_ERR_INVALID, "rows must be >= 1");
  if ((reinterpret_cast<uintptr_t>(x_f32) & 15u) || (reinterpret_cast<uintptr_t>(out_16bit) & 15u))
    return fail(SIGLIP_ERR_INVALID, "buffers must be 16-byte aligned");
  CK(cudaSetDevice(c->device));
  CKI(siglip::launch_convert_f32(x_f32, out_16bit, static_cast<size_t>(rows) * c->DT, f16 ? kXScale : 0.0f, c->num_sms,
                                 static_cast<cudaStream_t>(cuda_stream)));
  c->launches++;
  return 0;
}

int siglip_teacher_normalize_fwd(siglip_ctx* c, int rows, const void* x, int in_bf16, void* xhat, float* inv_norm,
                                 int f16, void* cuda_stream) {
  if (c == nullptr || x == nullptr || xhat == nullptr || inv_norm == nullptr)
    return fail(SIGLIP_ERR_INVALID, "null argument");
  if (c->DT == 0) return fail(SIGLIP_ERR_STATE, "not a distillation context (siglip_ctx_create_distill)");
  if (rows < 1) return fail(SIGLIP_ERR_INVALID, "rows must be >= 1");
  if ((reinterpret_cast<uintptr_t>(x) & 15u) || (reinterpret_cast<uintptr_t>(xhat) & 15u))
    return fail(SIGLIP_ERR_INVALID, "buffers must be 16-byte aligned");
  CK(cudaSetDevice(c->device));
  CKI(siglip::launch_normalize_fwd(x, in_bf16, static_cast<__nv_bfloat16*>(xhat), inv_norm, rows, c->DT,
                                   f16 ? kXScale : 0.0f, c->num_sms, static_cast<cudaStream_t>(cuda_stream)));
  c->launches++;
  return 0;
}

int siglip_debug_set_chunk_ids(siglip_ctx* c, int chunk, const int64_t* ids_dev, void* cuda_stream) {
  if (c == nullptr || ids_dev == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (c->world == 1 || chunk < 0 || chunk >= c->world) return fail(SIGLIP_ERR_INVALID, "chunk out of range");
  CK(cudaMemcpyAsync(c->ids_all + static_cast<size_t>(chunk) * ids_slot(c), ids_dev, chunk_ids_bytes(c, chunk),
                     cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(cuda_stream)));
  return 0;
}

int siglip_debug_set_chunk_groups(siglip_ctx* c, int chunk, const int64_t* groups_dev, void* cuda_stream) {
  if (c == nullptr || groups_dev == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (c->world == 1 || chunk < 0 || chunk >= c->world) return fail(SIGLIP_ERR_INVALID, "chunk out of range");
  // the group half of the chunk's slot, where its owner's ids publish puts them
  CK(cudaMemcpyAsync(c->ids_all + static_cast<size_t>(chunk) * ids_slot(c) + set_words(c), groups_dev,
                     static_cast<size_t>(c->Ts[chunk]) * sizeof(int64_t), cudaMemcpyDeviceToDevice,
                     static_cast<cudaStream_t>(cuda_stream)));
  return 0;
}

int siglip_debug_set_chunk_label_sets(siglip_ctx* c, int chunk, const int64_t* sets_dev, void* cuda_stream) {
  if (c == nullptr || sets_dev == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (c->world == 1 || chunk < 0 || chunk >= c->world) return fail(SIGLIP_ERR_INVALID, "chunk out of range");
  if (c->LM == 0) return fail(SIGLIP_ERR_STATE, "siglip_debug_set_chunk_label_sets needs a context with label sets");
  // the set half of the chunk's slot, where its owner's ids publish puts them
  CK(cudaMemcpyAsync(c->ids_all + static_cast<size_t>(chunk) * ids_slot(c), sets_dev,
                     static_cast<size_t>(c->Ts[chunk]) * c->LM * sizeof(int64_t), cudaMemcpyDeviceToDevice,
                     static_cast<cudaStream_t>(cuda_stream)));
  return 0;
}

int siglip_debug_set_chunk_weights(siglip_ctx* c, int chunk, const float* text_w_dev, void* cuda_stream) {
  if (c == nullptr) return fail(SIGLIP_ERR_INVALID, "ctx is null");
  if (c->world == 1 || chunk < 0 || chunk >= c->world) return fail(SIGLIP_ERR_INVALID, "chunk out of range");
  // clamped like the owner's siglip_set_sample_weights (NULL = ones)
  CKI(siglip::launch_clamp_weights(text_w_dev, c->w_all + static_cast<size_t>(chunk) * c->w_stride, c->Ts[chunk],
                                   nullptr, nullptr, 0, static_cast<cudaStream_t>(cuda_stream)));
  c->launches++;
  return 0;
}

int siglip_debug_get_slot(siglip_ctx* c, int chunk, float* out_dev, void* cuda_stream) {
  if (c == nullptr || out_dev == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (c->world == 1 || chunk < 0 || chunk >= c->world) return fail(SIGLIP_ERR_INVALID, "chunk out of range");
  CK(cudaMemcpyAsync(out_dev, c->slots + chunk * chunk_stride(c),
                     static_cast<size_t>(c->Ts[chunk]) * c->D * sizeof(float), cudaMemcpyDeviceToDevice,
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
  if (c == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  return siglip_normalize_fwd_rows(c, c->B, x, in_bf16, xhat_bf16, inv_norm, cuda_stream);
}

int siglip_normalize_fwd_rows(siglip_ctx* c, int rows, const void* x, int in_bf16, void* xhat_bf16, float* inv_norm,
                              void* cuda_stream) {
  if (c == nullptr || x == nullptr || xhat_bf16 == nullptr || inv_norm == nullptr)
    return fail(SIGLIP_ERR_INVALID, "null argument");
  if (rows < 1) return fail(SIGLIP_ERR_INVALID, "rows must be >= 1");
  if ((reinterpret_cast<uintptr_t>(x) & 15u) || (reinterpret_cast<uintptr_t>(xhat_bf16) & 15u))
    return fail(SIGLIP_ERR_INVALID, "buffers must be 16-byte aligned");
  CK(cudaSetDevice(c->device));
  CKI(siglip::launch_normalize_fwd(x, in_bf16, static_cast<__nv_bfloat16*>(xhat_bf16), inv_norm, rows, c->D,
                                   c->input_f16 ? kXScale : 0.0f, c->num_sms, static_cast<cudaStream_t>(cuda_stream)));
  c->launches++;
  return 0;
}

int siglip_convert_f32(siglip_ctx* c, const float* x_f32, void* out_16bit, void* cuda_stream) {
  if (c == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  return siglip_convert_f32_rows(c, c->B, x_f32, out_16bit, cuda_stream);
}

int siglip_convert_f32_rows(siglip_ctx* c, int rows, const float* x_f32, void* out_16bit, void* cuda_stream) {
  if (c == nullptr || x_f32 == nullptr || out_16bit == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  if (rows < 1) return fail(SIGLIP_ERR_INVALID, "rows must be >= 1");
  if ((reinterpret_cast<uintptr_t>(x_f32) & 15u) || (reinterpret_cast<uintptr_t>(out_16bit) & 15u))
    return fail(SIGLIP_ERR_INVALID, "buffers must be 16-byte aligned");
  CK(cudaSetDevice(c->device));
  CKI(siglip::launch_convert_f32(x_f32, out_16bit, static_cast<size_t>(rows) * c->D, c->input_f16 ? kXScale : 0.0f,
                                 c->num_sms, static_cast<cudaStream_t>(cuda_stream)));
  c->launches++;
  return 0;
}

int siglip_normalize_bwd(siglip_ctx* c, const void* x, int in_bf16, const float* inv_norm, const void* dxhat,
                         int grad_bf16, void* dx, void* cuda_stream) {
  if (c == nullptr) return fail(SIGLIP_ERR_INVALID, "null argument");
  return siglip_normalize_bwd_rows(c, c->B, x, in_bf16, inv_norm, dxhat, grad_bf16, dx, cuda_stream);
}

int siglip_normalize_bwd_rows(siglip_ctx* c, int rows, const void* x, int in_bf16, const float* inv_norm,
                              const void* dxhat, int grad_bf16, void* dx, void* cuda_stream) {
  if (c == nullptr || x == nullptr || inv_norm == nullptr || dxhat == nullptr || dx == nullptr)
    return fail(SIGLIP_ERR_INVALID, "null argument");
  if (rows < 1) return fail(SIGLIP_ERR_INVALID, "rows must be >= 1");
  if ((reinterpret_cast<uintptr_t>(x) & 15u) || (reinterpret_cast<uintptr_t>(dxhat) & 15u) ||
      (reinterpret_cast<uintptr_t>(dx) & 15u))
    return fail(SIGLIP_ERR_INVALID, "buffers must be 16-byte aligned");
  CK(cudaSetDevice(c->device));
  CKI(siglip::launch_normalize_bwd(x, in_bf16, inv_norm, dxhat, grad_bf16, dx, rows, c->D, c->num_sms,
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
  const char* env_tn = getenv("SIGLIP_DEBUG_TILE_N");
  const int tile_n = env_tn ? atoi(env_tn) : siglip::kTileCols;
  if (tile_n != siglip::kTileCols && tile_n != siglip::kWideTileCols)
    return fail(SIGLIP_ERR_INVALID, "SIGLIP_DEBUG_TILE_N must be 128 or 256");
  if (fp8 && tile_n != siglip::kTileCols) return fail(SIGLIP_ERR_INVALID, "the fp8 measurement path has 128-column tiles");
  if (fp8) {
    if (a_mn || b_mn || mcast != 1) return fail(SIGLIP_ERR_INVALID, "the fp8 measurement path is K-major, no multicast");
    if ((rc = encode_u8_kmajor(&tmA, A, M, K, lda, 128))) return rc;
    if ((rc = encode_u8_kmajor(&tmB, Bm, N, K, ldb, siglip::b_box_rows_kmajor(cta_group)))) return rc;
  } else {
    const int cs = siglip::cluster_size(cta_group, mcast);
    if ((rc = encode_operand(&tmA, A, M, K, lda, a_mn, 128))) return rc;
    if ((rc = encode_operand(&tmB, Bm, N, K, ldb, b_mn, siglip::b_box_rows_kmajor(cs, tile_n),
                             siglip::b_box_k_mnmajor(cs, tile_n))))
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
    lrc = siglip::launch_gemm(cta_group, siglip::kModeOut, stages, mcast, tile_n, &tmA, &tmB, &tmA, &tmB, &tmA, p,
                              num_sms, st);
  cudaEventRecord(e0, st);
  for (int it = 0; it < iters && lrc == 0; ++it)
    lrc = siglip::launch_gemm(cta_group, siglip::kModeOut, stages, mcast, tile_n, &tmA, &tmB, &tmA, &tmB, &tmA, p,
                              num_sms, st);
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
  cudaFree(c->ids_in);
  cudaFree(c->rids);
  cudaFree(c->iota);
  cudaFree(c->loop_xids);
  cudaFree(c->lrows);
  cudaFree(c->xid_ptrs_dev);
  cudaFree(c->w_in);   // w_all: part of txt_all
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
  cudaFree(c->loop_keys);
  if (c->world == 1) cudaFree(c->mkeys[0]);   // world > 1: part of txt_all
  cudaFree(c->mkey_ptrs_dev);
  cudaFree(c->loop_lsums);
  if (c->world == 1) cudaFree(c->lsum[0]);    // world > 1: part of txt_all
  cudaFree(c->lsum_ptrs_dev);
  cudaFree(c->loop_topk);
  cudaFree(c->tk_rows[0]);                    // allocated by the first request (world == 1: with the column lists)
  cudaFree(c->tk_ptrs_dev);
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
