// Host-visible declarations of the sm_90a kernels (definitions in siglip_kernels.cu).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ptx.cuh"

namespace siglip {

// One dense contraction C[M,N] = A[M,K] * B[N,K]^T on the wgmma tensor cores, in 128 x 128 tiles (one per CTA).
// `a_mn` / `b_mn` say how the operand sits in memory:
//   0: K-major  — global tensor is [rows][K], K contiguous      (TMA box {64 k, rows}: A 128 rows, B kTileN / cluster)
//   1: MN-major — global tensor is [K][rows], rows contiguous   (TMA boxes {64 rows, 64 k}; B of a 4-CTA cluster {64, 32})
struct Problem {
  int M, N, K;
  int tiles_m, tiles_n;   // filled in by launch_gemm: row panels of one cluster, column tiles (128 or 256 wide)
  int a_mn, b_mn;
  int ab_f16;       // 0: bf16 operands; 1: both IEEE fp16 (gradient contractions: scaled sigma x scaled embeddings);
                    // 2: both fp8 e4m3, K-major only (the SURVEY.md §8f-4 measurement, siglip_debug_gemm)
  float acc_scale;  // multiplies the accumulator in the out epilogue (2^-k for a 2^k-scaled fp16 A operand)
  // epilogue of the "out" kernel:
  //   out = scale * (acc * acc_scale + fix_vec[row] * fix_mat[row, col]) (+ add_src[row, col]); fp32 or bf16 output
  void* out;
  long long ldo;
  int out_bf16;
  const float* fix_vec;
  const __nv_bfloat16* fix_mat;   // bf16 values, or (fix_f16) IEEE fp16 values scaled by 1 / fix_mat_scale
  long long ldx;
  int fix_f16;
  float fix_mat_scale;    // multiplies the decoded fix_mat value (1/16 for the fp16 x 16 embeddings; 0 = 1)
  const float* add_src;   // optional fp32 term (running dimg of the previous chunks)
  long long ld_add;
};

constexpr int kMaxAuxJobs = 8;   // L0 of a multi-rank step with sample ids carries 7, with ids and weights 8
                                 // (DESIGN.md, "Per-sample loss weights")
enum AuxKind { kAuxNone = 0, kAuxCopy = 1, kAuxCvt = 2, kAuxFold = 3, kAuxWaitOnly = 4 };

// One job of the auxiliary warps. Optional pre-wait on `wait_n` consecutive local flags (all >= wait_value, written by
// peers with st.release.sys), then the data movement, then — once EVERY CTA has finished its share (ticket) — an
// optional release-store of sig_value to sig_n peer flags and / or of done_value to a local flag.
struct AuxJob {
  int kind;
  const volatile unsigned int* wait_flags;  // null = no wait
  int wait_n;
  unsigned int wait_value;
  unsigned int site;          // id reported if the wait times out
  const uint4* src;           // kAuxCopy / kAuxCvt: source (may be peer memory); kAuxFold: remote fp32 contribution
  const uint4* src2;          // kAuxFold: local fp32 accumulator input (null = 0)
  uint4* dst;
  unsigned long long n16;     // 16-byte vectors
  int cvt_copy;               // kAuxCvt: 1 = plain copy (sources already fp16)
  unsigned int* const* sig_ptrs;
  int sig_n;
  unsigned int sig_value;
  unsigned int* done_flag;    // local flag (gpu scope) set to done_value when the job is complete on every CTA
  unsigned int done_value;
  unsigned int* ticket;       // zero between launches; required when sig_n > 0 or done_flag != null
};

struct KernelParams {
  Problem prob[2];
  int nprob;
  // learnable scalars, device memory (reference: distributed_sigmoid_loss.py:11-12)
  const float* t_prime;   // fp32, or fp64 when tprime_f64 (then sc_dt_prime is written as fp64 too)
  int tprime_f64;
  const float* bias;
  float s_scale;  // loss kernel: accumulator -> <img, txt> (2^-8 when both operands are fp16 x 16; 0 = 1)
  float inv_b;  // 1 / per-rank batch (reference divides by the LOCAL batch, distributed_sigmoid_loss.py:47)
  const float* grad_out;  // out kernel: optional device scalar multiplied into every gradient (autograd's grad_output)
  // epilogue of the "loss" kernel
  __nv_bfloat16* G;  // [Bp, ldg] 16-bit sigma terms (fp16 bits, x g_scale), diagonal zeroed; may be null when store_g == 0
  long long ldg;
  float* g_diag;   // [B] fp32: -sigma(-z_ii), the positive-pair term kept out of the 16-bit operand
  int own_chunk;   // 1: this text chunk holds the positives of this rank's images
  int store_g;     // 0: forward only
  float g_scale;   // sigma is stored as fp16(sigma * g_scale): 2^14 keeps sigma in (3.7e-9, 1) inside fp16's normal range
  // sample-id labels (SIGLIP_OPT_SAMPLE_IDS): pair (i, j) is positive iff row_ids[i] == col_ids[j]. row_ids: this rank's
  // images [M]; col_ids: the text chunk being scored [N]. Null = positional labels (the own-chunk diagonal only).
  const int64_t* row_ids;
  const int64_t* col_ids;
  double* partials;  // [gridDim.x][4] : sum softplus, sum g, sum g*s, (unused)
  int accumulate_partials;
  // loss kernel of the LAST chunk of a forward: the CTA that finishes last (ticket counter) adds the per-CTA slots in
  // slot order and writes loss (and, when saving for backward, dt' / dbias for an upstream gradient of 1)
  unsigned int* fin_counter;   // null = no finalisation in this launch
  float* fin_loss;
  float* fin_dt_prime;         // may be null
  float* fin_dbias;            // may be null
  // gradient kernel: dt' / dbias of the backward = saved value * grad_out, written by one thread (null = skip)
  const float* sc_saved;       // [2]
  float* sc_dt_prime;
  float* sc_dbias;
  DebugRecord* dbg;
  unsigned long long* wait_stats;  // optional [gridDim.x][4]: producer empty-wait, MMA full-wait, MMA tmem-wait, MMA loop cycles
  // Work of the two auxiliary warps of every CTA while the tiles compute: up to kMaxAuxJobs jobs executed in order,
  // each spread over all CTAs of the launch (grid-stride over 16-byte vectors). This is where the cross-rank exchange
  // lives: peer pulls of text chunks and folds of the peers' dtxt contributions over NVSwitch P2P, ordered by flags.
  AuxJob aux[kMaxAuxJobs];
  int naux;
  float cvt_scale;   // kAuxCvt: dst = fp16(src_bf16 * cvt_scale), clamped
  // Signal written when the LAST CTA of the launch has finished (ticket counter): everything this launch wrote is then
  // visible to the peers that observe the flag (st.release.sys after a system-scope fence).
  unsigned int* const* end_sig_ptrs;   // device array of flag addresses (peer-mapped), null = no signal
  int end_sig_n;
  unsigned int end_sig_value;
  unsigned int* end_ticket;
  // out kernel, problem 1: do not read add_src before this local flag (set by an aux job's done_flag) holds done_value
  const volatile unsigned int* p1_wait_flag;
  unsigned int p1_wait_value;
  // Split-K of the ragged last wave (out kernel, no multicast): work items [sk_first, sk_first + sk_tiles * sk_parts)
  // are K-slices of the last sk_tiles tiles; slice 0 owns the tile: it waits for the others' fp32 partial accumulators
  // in sk_ws and adds them in slice order (bitwise independent of timing).
  int sk_parts;                // 0 / 1 = off
  int sk_first;
  int sk_tiles;
  int sk_request;              // host request to launch_gemm: -1 choose, 0 off, S >= 2
  float* sk_ws;                // [sk_tiles][sk_parts - 1][cluster CTA][128 x 128 fp32 in fragment order]
  size_t sk_ws_bytes;
  unsigned int* sk_counters;   // [sk_tiles][2]: arrivals of the non-owner warps, owner warps that consumed them
  int sk_max_tiles;            // capacity of sk_counters
  int pdl;                     // 1: launched with programmatic stream serialization (griddepcontrol in the kernel)
  unsigned long long peer_timeout_ns;  // bound of every wait on a peer flag (a dead peer traps instead of hanging)
  unsigned long long* aux_trace;       // optional [4] globaltimer stamps of CTA 0's aux thread: start, flags seen, jobs done
  // In-batch retrieval metrics (siglip_request_metrics), loss kernel only. Appended last so that the parameter offsets of
  // the default instantiation do not move. Non-null keys select the kMetrics instantiation. A key is
  // (order-preserving bits of s) << 32 | (0xFFFFFFFF - global index), combined with an atomic unsigned max: the best
  // candidate, ties to the lowest index, independent of the order of the atomics.
  unsigned long long* row_keys;  // [M]: best text (global index) of each image of this rank
  unsigned long long* col_keys;  // [N]: best image (global index) of each text of the chunk, over this rank's images
  int row_off;                   // global index of this rank's first image
  int col_off;                   // global index of the chunk's first text
  // Hard-negative captions (siglip_ctx_create_texts): a text chunk is [paired texts; extras]. Appended last like the
  // metrics fields, so that the default loss kernel's parameter offsets do not move.
  int col_pos_n;   // loss kernel, kIds: columns of the chunk that carry ids (col_ids has this many entries): its paired
                   // texts, or all of them under SIGLIP_OPT_EXTRA_TEXT_IDS. Columns past it never match
  int fix_rows;    // out kernel: rows of fix_vec / fix_mat (this rank's batch); rows >= fix_rows take no fix term
  // Host only (launch_gemm): size the grid of a loss launch as if its chunk had grid_n columns. Every loss kernel of a
  // forward then has the same grid, so the per-CTA partial slots it accumulates and the last one sums line up when the
  // chunks have different sizes (uneven batches, hard negatives). 0 = the chunk's own N.
  int grid_n;
  // Per-sample loss weights (SIGLIP_OPT_SAMPLE_WEIGHTS), loss kernel only. Appended last like the fields above. Non-null
  // row_w selects the kWeights instantiation: pair (i, j) contributes w_ij = row_w[i] * col_w[j] times its softplus and
  // sigma terms, to the three sums, to g_diag and to the stored sigma operand. Both in [0, 1] (clamped on the way in).
  const float* row_w;   // [M]: this rank's image weights
  const float* col_w;   // [N]: weights of the texts of the chunk being scored
  // Extra images (siglip_ctx_create_extras): the rows are [paired images; extras]. Appended last like the fields above,
  // and read only by the kIds instantiations: the row twin of col_pos_n.
  int row_pos_n;   // loss kernel, kIds: rows that carry ids (row_ids has this many entries): the paired images, or all
                   // of them under SIGLIP_OPT_EXTRA_IMAGE_IDS. Rows past it never match
  // Distillation from a frozen teacher (siglip_set_teacher). Appended last like the fields above. k_teacher > 0 selects
  // the distillation loss kernel (kModeDistill, its own instantiation): every tile first contracts the teacher's image
  // rows (tmA1) with the teacher's text chunk (tmB1) over k_teacher, turns s^T into p = sigma(t_T s^T + b_T), then runs
  // the student's k-loop; the target of pair (i, j) is q = (1 - lambda) y + lambda p. In that kernel ids (row_ids),
  // weights (row_w) and metric keys (row_keys) are runtime options. With sl_rows, tk_rows, col_grp or col_lab set as
  // well, the launch runs kModeDistillOpts, which takes all of those as runtime options too.
  int k_teacher;              // D_T (multiple of 8); 0 = no teacher
  int teacher_f16;            // teacher operands are fp16(x * 16) instead of bf16
  const float* t_prime_T;     // fp32 device scalars: t_T = exp(t'_T), b_T
  const float* bias_T;
  float distill_lambda;       // in (0, 1]
  // Per-sample losses (siglip_request_sample_losses). Appended last like the fields above. Non-null sl_rows selects the
  // kModeSampleLoss loss kernel: besides the three sums it adds every tile's row sums and every 16-row slab's column
  // sums of the terms w_ij softplus(-y_ij z_ij) into 64-bit fixed-point words (value * 2^32, red.add.u64), so that the
  // result does not depend on the order of the atomics. A partial that is not finite or >= kSampleLossMaxPartial ORs a
  // poison bit (1: too large or +inf, 2: NaN) into the word sl_poison words behind its sum instead.
  unsigned long long* sl_rows;   // [M]: sums of this rank's images over the chunk's texts
  unsigned long long* sl_cols;   // [N]: sums of the chunk's texts over this rank's images
  long long sl_poison;           // distance in words from a sum to its poison word
  // Top-K retrieval (siglip_request_topk, K > 1). Appended last like the fields above. Non-null tk_rows selects the
  // kModeTopK loss kernel: besides the kModeSampleLoss epilogue (whose sums are then optional) it inserts every
  // candidate key above a list's current K-th entry into that row's / column's sorted list of kTopKMax slots with a
  // chain of atomic maxima (tile_topk). Keys as row_keys / col_keys, global indices from row_off / col_off.
  unsigned long long* tk_rows;   // [M][kTopKMax]: the best texts of each image of this rank
  unsigned long long* tk_cols;   // [N][kTopKMax]: the best images of each text of the chunk, over this rank's images
  int tk_k;                      // K in 2 .. kTopKMax: slots of each list that are filled
  // Excluded pairs from group ids (SIGLIP_OPT_EXCLUDE_GROUPS). Appended last like the fields above. Non-null col_grp
  // selects the kModeGroups loss kernel: a pair (i, j) that is not a positive and whose groups match
  // (row_grp[i] == col_grp[j] >= 0) contributes 0 to the sums, the sigma operand and the per-sample sums.
  const int64_t* row_grp;        // [grp_rows]: groups of this rank's images (rows of the launch)
  const int64_t* col_grp;        // [N]: groups of the texts of the chunk being scored
  int grp_rows;                  // rows that carry a group (row_grp has this many entries); rows past it match nothing
  // Multi-label positives from label sets (SIGLIP_OPT_LABEL_SETS). Appended last like the fields above. Non-null
  // col_lab selects the kModeLabels loss kernel: a pair (i, j) is also a positive when the sets row_lab[i] and col_lab[j]
  // share a label >= 0 (negative entries are empty slots). Groups, ids, weights, metric keys, per-sample sums and top-K
  // lists stay runtime options there; excluded groups apply after these positives.
  const int64_t* row_lab;        // [M][lab_m]: the sets of this rank's images (rows of the launch)
  const int64_t* col_lab;        // [N][lab_m]: the sets of the texts of the chunk being scored
  int lab_m;                     // labels per set, 1 .. kMaxLabels
  // Focal pair loss (SIGLIP_OPT_FOCAL, siglip_set_focal). Appended last like the fields above. focal != 0 selects the
  // kModeFocal loss kernel: pair (i, j) with target y, p = sigma(z), p_t = y ? p : 1 - p and a_t = y ? alpha : 1 - alpha
  // (1 without alpha) adds a_t (1 - p_t)^gamma softplus(-(2y - 1) z) and stores its derivative in z. Ids, label sets,
  // weights, excluded groups, metric keys, per-sample sums and top-K lists stay runtime options there.
  int focal;
  float focal_gamma;             // in [0, 8]
  float focal_alpha;             // in [0, 1]; < 0: no alpha (a_t = 1)
};

// kModeDistill: the loss kernel of a distillation step (KernelParams::k_teacher > 0), its own instantiation
// kModeSampleLoss: the loss kernel of a step with per-sample losses (KernelParams::sl_rows != null), its own
// instantiation; ids, weights and metric keys are runtime options in it
// kModeTopK: the loss kernel of a top-K step (KernelParams::tk_rows != null), its own instantiation; ids, weights,
// metric keys and per-sample-loss sums are runtime options in it
// kModeGroups: the loss kernel of a step with excluded same-group pairs (KernelParams::col_grp != null), its own
// instantiation; ids, weights, metric keys, per-sample-loss sums and top-K lists are runtime options in it
// kModeLabels: the loss kernel of a step with label sets (KernelParams::col_lab != null), its own instantiation; ids,
// weights, metric keys, per-sample-loss sums, top-K lists and excluded groups are runtime options in it
// kModeFocal: the loss kernel of a focal step (KernelParams::focal != 0), its own instantiation; ids, label sets,
// weights, metric keys, per-sample-loss sums, top-K lists and excluded groups are runtime options in it
// kModeDistillOpts: the loss kernel of a distillation step with per-sample losses, top-K lists, excluded groups or label
// sets (k_teacher > 0 and any of sl_rows, tk_rows, col_grp, col_lab), its own instantiation; the teacher pass of
// kModeDistill, then the soft-target terms in the kModeFocal epilogue; ids, label sets, weights, excluded groups, metric
// keys, per-sample-loss sums and top-K lists are runtime options in it
enum KernelMode {
  kModeLoss = 0,
  kModeOut = 1,
  kModeDistill = 2,
  kModeSampleLoss = 3,
  kModeTopK = 4,
  kModeGroups = 5,
  kModeLabels = 6,
  kModeFocal = 7,
  kModeDistillOpts = 8
};

// Label sets: labels per set at most (SIGLIP_MAX_LABELS)
constexpr int kMaxLabels = 4;

// Top-K retrieval: slots of every list (SIGLIP_TOPK_MAX), whatever K the step asks
constexpr int kTopKMax = 10;

// Per-sample losses: fixed-point scale of the 64-bit sums, and the largest partial (one tile's row sum over 128
// columns, or one 16-row slab's column sum) that is added as a number. 2^16 * 2^32 per partial keeps the unsigned sum
// of up to 2^16 partials per sample (a global batch of up to 2^20 images and 2^23 texts) inside 64 bits.
constexpr double kSampleLossScale = 4294967296.0;        // 2^32
constexpr float kSampleLossMaxPartial = 65536.0f;        // 2^16

// Pipeline depth of the distillation loss kernel: 4 stages of 32 KiB leave room for the 64 KiB of teacher
// probabilities (fp32, 128 x 128 per CTA) next to the sigma staging buffers.
constexpr int kDistillStages = 4;

constexpr int kTileCols = 128;   // columns of a tile (wgmma N); a CTA computes 128 rows of it
constexpr int kWideTileCols = 256;   // the gradient kernel's wide tiles (out mode, 16-bit operands, no split-K)

// CTAs per cluster: cta_group (1 or 2) CTAs compute one 128- or 256-row tile, mcast (1 or 2) such tiles share their B
// tile as well; either way a cluster is a column of vertically adjacent 128-row blocks sharing B through TMA multicast.
inline int cluster_size(int cta_group, int mcast) { return cta_group * mcast; }
// Box of the B operand's tensor map for a cluster of `cs` CTAs and tiles `tile_n` columns wide (each CTA fetches
// 1 / cs of the B tile): K-major rows, MN-major k extent. MN-major boxes are 64 columns wide: a 128-column tile of a
// 4-CTA cluster is fetched in k halves, every other tile in whole {64, 64} boxes.
inline int b_box_rows_kmajor(int cs, int tile_n = kTileCols) { return tile_n / cs; }
inline int b_box_k_mnmajor(int cs, int tile_n = kTileCols) { return (cs == 4 && tile_n == kTileCols) ? 32 : 64; }

// Dynamic shared memory needed by the default configuration of `mode`.
size_t gemm_smem_bytes(int mode);
int default_stages(int mode);
// Clusters of the persistent grid of the out kernel with `cluster` CTAs per cluster, tile_n columns (kTileCols or
// kWideTileCols) and `stages` (4, else 6; the wide tiles always have kWideStages): what launch_impl launches
// (diagnostics and tests). -1 without a device.
int query_max_active_clusters(int cluster, int tile_n = kTileCols, int stages = 6);
// The same for the loss kernel of `mode` (kModeLoss or one of its twins; stages 4, else 6; the teacher modes always have
// kDistillStages). -1 without a device, -2 for a mode that is not a loss mode.
int query_loss_max_active_clusters(int mode, int cluster, int stages);

// Launch the warp-specialised persistent kernel. `stages` <= 0 selects the default pipeline depth (4 or 6).
// tmG: store map of the sigma operand (loss mode; 16-bit [B, B], box {32, 16}, 64B swizzle) — any valid map in out mode.
// Returns cudaError_t as int.
// cta_group x mcast = CTAs per cluster (1, 2 or 4); the B maps must have the boxes b_box_rows_kmajor /
// b_box_k_mnmajor give for that cluster size and tile width.
// tile_n: kTileCols, or kWideTileCols for the out kernel with 16-bit operands (4 stages whatever `stages` asks; never
// split along K). Anything else is cudaErrorInvalidValue.
int launch_gemm(int cta_group, int mode, int stages, int mcast, int tile_n, const CUtensorMap* tmA0,
                const CUtensorMap* tmB0, const CUtensorMap* tmA1, const CUtensorMap* tmB1, const CUtensorMap* tmG,
                const KernelParams& p, int num_sms, cudaStream_t stream);

// loss = inv_b * S0 ; dbias = inv_b * S1 ; dt_prime = exp(t') * inv_b * S2  (S* = fixed-order sums of partials)
// dtxt[j, d] = sum_r slots[r][j, d]   (slots may be peer-mapped pointers; fp32; n = elements)
int launch_reduce_slots(void* out, int out_bf16, const float* const* slots_dev, int nslots, size_t n, int num_sms,
                        cudaStream_t stream);

// xhat = bf16(x / max(||x||, 1e-12)) row-wise, inv_norm[r] = 1 / max(||x_r||, 1e-12); x is fp32 or bf16 [rows, D]
int launch_normalize_fwd(const void* x, int in_bf16, __nv_bfloat16* xhat, float* inv_norm, int rows, int D,
                         float f16_scale, int num_sms, cudaStream_t stream);
int launch_convert_f32(const float* src, void* dst, size_t n, float f16_scale, int num_sms, cudaStream_t stream);
// dx = inv_norm * (dxhat - xhat <xhat, dxhat>), xhat recomputed in fp32 from x; dx has x's dtype
int launch_normalize_bwd(const void* x, int in_bf16, const float* inv_norm, const void* dxhat, int grad_bf16, void* dx,
                         int rows, int D, int num_sms, cudaStream_t stream);

// dst = src * (*g) over nbytes (multiple of 16) of fp32 or bf16 data
int launch_scale(const void* src, void* dst, int is_bf16, const float* g, size_t nbytes, int num_sms,
                 cudaStream_t stream);

// cross-rank flag helpers (peer-mapped pointers)
int launch_allreduce_scalars(const float* saved, const float* g, float* mailbox_local, const float* const* mailboxes_dev,
                             unsigned int* const* signal_ptrs_dev, const volatile unsigned int* flags_local, int world,
                             unsigned int value, float* dt_prime, float* dbias, int dtp_f64,
                             unsigned long long timeout_ns, DebugRecord* dbg, cudaStream_t stream);
int launch_signal_flags(unsigned int* const* flag_ptrs_dev, int n, unsigned int value, cudaStream_t stream);

// Finalisation of a metrics step (one block, after the step's last loss kernel). W > 1: publish "my column partials of
// step `value` are complete" (flag kind 5) to every rank, wait for every rank's, and max-combine the W partials of my
// chunk. Then decode the keys into global indices and count the hits (positional, or same sample id).
constexpr int kMetricsMaxWorld = 32;
struct MetricsArgs {
  const unsigned long long* row_keys;          // [B] local
  const unsigned long long* col_own;           // [T] my partial of my chunk
  const unsigned long long* const* col_peers;  // [world] every rank's partial of my chunk (world > 1; own entry unused)
  int B, rank, world;
  int off[kMetricsMaxWorld + 1];               // prefix sums of the per-rank image counts (global image indices): rank
                                               // p's images off[p] .. off[p] + B_p - 1 are paired, the rest extras
  int toff[kMetricsMaxWorld + 1];              // prefix sums of the per-rank text counts (global text indices): rank
                                               // p's texts toff[p] .. toff[p] + B_p - 1 are paired, the rest extras
  int bs[kMetricsMaxWorld];                    // per-rank batches B_p (paired images / texts)
  int R;                                       // this rank's images (B + its extra images)
  int extra_image_ids;                         // SIGLIP_OPT_EXTRA_IMAGE_IDS: i2t covers all R images (i2t: [R]) and a
                                               // winning extra image is a t2i hit when its id is the text's
  const int64_t* row_ids;                      // [R] ids of this rank's images (ids mode): the sample ids, then the
                                               // extra images' ids
  const int64_t* const* xids_peers;            // [world] every rank's published extra-image ids of this step (world > 1
                                               // under extra_image_ids; own entry unused)
  const int64_t* ids_own;                      // null = positional labels; else this rank's sample ids
  const int64_t* ids_all;                      // [world][ids_stride]: every chunk's ids, gathered in this step
  int ids_stride;
  int extra_ids;                               // SIGLIP_OPT_EXTRA_TEXT_IDS: every text has an id (ids_own: [T]),
                                               // extras can be hits, and t2i covers all T texts of this rank
  int T;                                       // this rank's texts
  float* top1;                                 // [2]: i2t, t2i
  int64_t* i2t;                                // [B] ([R] under extra_image_ids) or null
  int64_t* t2i;                                // [B] ([T] under extra_ids) or null
  unsigned int* const* sig_ptrs;               // [world] flag kind 5 of every rank (world > 1)
  const volatile unsigned int* flags_local;    // my flag kind 5 row
  unsigned int value;
  unsigned long long timeout_ns;
  DebugRecord* dbg;
};
int launch_metrics_finalize(const MetricsArgs& a, cudaStream_t stream);

// Finalisation of a per-sample-loss step (one block, after the step's last loss kernel, and after the metrics
// finalisation when both are armed). W > 1: unless the metrics finalisation already did, publish flag kind 5 to every
// rank; then wait for every rank's flag kind 5 of the step and add the W ranks' fixed-point partials of my chunk in rank
// order (relaxed system-scope loads). Decode rows into image_loss [R] and columns into text_loss [T].
struct SampleLossArgs {
  const unsigned long long* rows;              // [R] local row sums (poison words sl_poison words behind)
  const unsigned long long* col_own;           // [T] my partial of my chunk
  const unsigned long long* const* col_peers;  // [world] every rank's partial of my chunk (world > 1; own entry unused)
  long long poison;                            // distance in words from a sum to its poison word (same on every rank)
  int R, T, rank, world;
  int signal;                                  // 1: raise flag kind 5 here (no metrics finalisation in this step)
  float* image_loss;
  float* text_loss;
  unsigned int* const* sig_ptrs;               // [world] flag kind 5 of every rank (world > 1)
  const volatile unsigned int* flags_local;    // my flag kind 5 row
  unsigned int value;
  unsigned long long timeout_ns;
  DebugRecord* dbg;
};
int launch_sample_loss_finalize(const SampleLossArgs& a, cudaStream_t stream);

// Finalisation of a top-K step with K > 1 (one block, after the metrics finalisation when both are armed, before the
// per-sample losses). W > 1: unless the metrics finalisation already did, publish flag kind 5 to every rank; then wait
// for every rank's flag kind 5 of the step and merge the W sorted column lists of each of my texts (relaxed
// system-scope loads). Decode the lists into global indices and count, per side, the samples whose first hit is at
// each rank, for recall@k. m carries the hit rules and the flags as for the metrics (its key pointers are unused).
struct TopKArgs {
  MetricsArgs m;
  const unsigned long long* rows;              // [R][kTopKMax] local row lists
  const unsigned long long* col_own;           // [T][kTopKMax] my lists of my chunk
  const unsigned long long* const* col_peers;  // [world] every rank's lists of my chunk (world > 1; own entry unused)
  int k;
  int signal;                                  // 1: raise flag kind 5 here (no metrics finalisation in this step)
  float* recall;                               // [2k]: i2t, then t2i
  int64_t* i2t;                                // [ni][k] or null
  int64_t* t2i;                                // [nt][k] or null
};
int launch_topk_finalize(const TopKArgs& a, cudaStream_t stream);

// The hit rule of a label-set step (SIGLIP_OPT_LABEL_SETS) for the metrics and top-K finalisations: a hit is the
// positional pair (my image i and my paired text i, i < B) or a pair whose sets share a label >= 0. i2t ranks all R
// images and t2i all T texts. These launches run their own instantiation of the finalisation kernels; the MetricsArgs
// id fields are unused.
struct LabelSetArgs {
  const int64_t* row_sets;                     // [R][m] the sets of this rank's images: paired, then extra
  const int64_t* text_own;                     // [T][m] the sets of this rank's texts: paired, then extra
  const int64_t* text_all;                     // [world][slot]: every chunk's text sets, gathered in this step
  long long slot;                              // words between two chunks' sets in text_all
  const int64_t* const* xsets_peers;           // [world] every rank's published extra-image sets ([E_o][m]) of this
                                               // step (world > 1 with extra images; own entry unused)
  int m;                                       // labels per set
};
int launch_metrics_finalize_labels(const MetricsArgs& a, const LabelSetArgs& l, cudaStream_t stream);
int launch_topk_finalize_labels(const TopKArgs& a, const LabelSetArgs& l, cudaStream_t stream);
int launch_wait_flags(const volatile unsigned int* flags, int n, unsigned int value, unsigned long long timeout_ns,
                      DebugRecord* dbg, cudaStream_t stream);

// SIGLIP_OPT_SAMPLE_WEIGHTS: dst_a[0, na) = clamp(src_a) and dst_b[0, nb) = clamp(src_b) in one launch, where
// clamp(x) = min(max(x, 0), 1) and NaN -> 0; a null source gives ones.
int launch_clamp_weights(const float* src_a, float* dst_a, int na, const float* src_b, float* dst_b, int nb,
                         cudaStream_t stream);

}  // namespace siglip
