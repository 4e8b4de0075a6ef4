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
  int tiles_m, tiles_n;   // filled in by launch_gemm: row panels of one cluster, 128-column tiles
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

constexpr int kMaxAuxJobs = 6;
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
};

enum KernelMode { kModeLoss = 0, kModeOut = 1 };

constexpr int kTileCols = 128;   // columns of a tile (wgmma N); a CTA computes 128 rows of it

// CTAs per cluster: cta_group (1 or 2) CTAs compute one 128- or 256-row tile, mcast (1 or 2) such tiles share their B
// tile as well; either way a cluster is a column of vertically adjacent 128-row blocks sharing B through TMA multicast.
inline int cluster_size(int cta_group, int mcast) { return cta_group * mcast; }
// Box of the B operand's tensor map for a cluster of `cs` CTAs (each CTA fetches 1 / cs of the B tile):
// K-major rows, MN-major k extent.
inline int b_box_rows_kmajor(int cs) { return kTileCols / cs; }
inline int b_box_k_mnmajor(int cs) { return cs == 4 ? 32 : 64; }

// Dynamic shared memory needed by the default configuration of `mode`.
size_t gemm_smem_bytes(int mode);
int default_stages(int mode);
int query_max_active_clusters(int cluster);  // co-resident clusters of the out kernel (diagnostic)

// Launch the warp-specialised persistent kernel. `stages` <= 0 selects the default pipeline depth (4 or 6).
// tmG: store map of the sigma operand (loss mode; 16-bit [B, B], box {32, 16}, 64B swizzle) — any valid map in out mode.
// Returns cudaError_t as int.
// cta_group x mcast = CTAs per cluster (1, 2 or 4); the B maps must have the boxes b_box_rows_kmajor /
// b_box_k_mnmajor give for that cluster size.
int launch_gemm(int cta_group, int mode, int stages, int mcast, const CUtensorMap* tmA0, const CUtensorMap* tmB0,
                const CUtensorMap* tmA1, const CUtensorMap* tmB1, const CUtensorMap* tmG, const KernelParams& p,
                int num_sms, cudaStream_t stream);

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
int launch_wait_flags(const volatile unsigned int* flags, int n, unsigned int value, unsigned long long timeout_ns,
                      DebugRecord* dbg, cudaStream_t stream);

}  // namespace siglip
