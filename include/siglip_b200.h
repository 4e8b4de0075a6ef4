/*
 * siglip_b200.h — C ABI of the H100-native (sm_90a) distributed sigmoid (SigLIP) loss hot path.
 *
 * The reference (ahmdtaha/distributed_sigmoid_loss) has no FFI layer: its boundary is the Python
 * nn.Module `DDPSigmoidLoss.forward(image_embeddings, text_embeddings)` (distributed_sigmoid_loss.py:8-48)
 * plus torch.distributed collectives. Each entry point below names the reference code it replaces.
 * The library never allocates or frees caller memory, never throws; every call returns 0 on success or a
 * non-zero status whose text is available from siglip_last_error(). All device work is enqueued on the
 * caller's stream (pass torch.cuda.current_stream().cuda_stream); nothing here synchronises the host
 * except ctx create/destroy and handle import.
 *
 * Data layout: `img`, `txt` are row-major [B, D] bf16 device buffers, 16-byte aligned, D % 8 == 0.
 * `dimg`, `dtxt` are row-major [B, D] fp32 (or bf16 with SIGLIP_OPT_GRAD_BF16). Scalars are fp32 device scalars.
 */
#ifndef SIGLIP_B200_H_
#define SIGLIP_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct siglip_ctx siglip_ctx;

enum {
  SIGLIP_OK = 0,
  SIGLIP_ERR_INVALID = 1,   /* bad argument / shape (reference: broadcast RuntimeError when B != gpu_batch_size) */
  SIGLIP_ERR_CUDA = 2,      /* a CUDA runtime / driver call failed */
  SIGLIP_ERR_NO_DEVICE = 3, /* no sm_90 device: there is NO CPU fallback */
  SIGLIP_ERR_STATE = 4      /* call sequence error (e.g. world > 1 without imported peer handles) */
};

/*
 * Diagnostics read from the environment (never needed in production):
 *   SIGLIP_DEBUG_LOSS_WAITSTATS  print per-role wait / loop cycle counts of every loss-kernel launch (synchronises)
 *   SIGLIP_DEBUG_NO_GSTORE, SIGLIP_DEBUG_NO_CVT   timing experiments: skip the sigma store / the fp16 operand copies
 *                                (the gradients are then WRONG)
 *   SIGLIP_DEBUG_PRINT_TIMES     print the per-launch CUDA-event times collected under SIGLIP_OPT_KERNEL_TIMING
 *   SIGLIP_DEBUG_MCAST, _AB_F16, _AB_FP8, _WAITSTATS, _STAGES   variants of siglip_debug_gemm(_timed) only
 */

/* tuning knobs (siglip_ctx_set_option) */
enum {
  SIGLIP_OPT_CTA_GROUP = 1, /* 1: every CTA computes its own 128-row tile; 2 (default): clusters of two CTAs on adjacent
                               128-row blocks share the B tile by TMA multicast. Tiles are 128 columns wide */
  SIGLIP_OPT_OVERLAP_PULL = 2, /* 1 (default): pull the next text chunk inside the loss kernel; 0: separate copy */
  SIGLIP_OPT_KERNEL_TIMING = 3, /* 1: bracket every loss / gradient kernel launch with CUDA events on the caller's stream */
  SIGLIP_OPT_STAGES_LOSS = 4,  /* TMA->MMA pipeline depth of the loss kernel: 0 (default, = 6), 4 or 6 */
  SIGLIP_OPT_STAGES_GRAD = 5,  /* ... of the gradient kernel */
  SIGLIP_OPT_MCAST = 6,        /* 2: twice as many vertically adjacent CTAs share the B tile by TMA multicast (cta_group 2:
                                  clusters of 4); default 1 */
  SIGLIP_OPT_GRAD_BF16 = 7,     /* 1: siglip_fwd_bwd writes dimg / dtxt as bf16 [B, D] (the dtype autograd returns for bf16 inputs); default 0 = fp32 */
  SIGLIP_OPT_OVERLAP_REDUCE = 8, /* 1 (default): fold the peers' dtxt contributions in step by step inside the gradient kernels; 0: one reduction at the end */
  SIGLIP_OPT_EPI_SLEEP_GRAD_NS = 9, /* accepted, no effect on sm_90a: the warps that run the epilogue also issue the MMAs
                                       and never wait idle for an accumulator (gradient kernel) */
  SIGLIP_OPT_EPI_SLEEP_LOSS_NS = 10, /* ... (loss kernel) */
  SIGLIP_OPT_SYNC_SCALAR_GRADS = 11, /* 1: siglip_backward returns the MEAN over ranks of dt_prime / dbias (what DDP's
                                        all-reduce of the two parameters does, README.md:20,
                                        test_distributed_sigmoid_loss.py:79-83), exchanged through peer memory by a
                                        one-warp kernel; bit-identical on every rank. Collective: set on all ranks */
  SIGLIP_OPT_BIDIR = 12, /* 1: visit the text chunks in the order r, r+1, r-1, r+2, r-2, ... (the order of the reference's
                            bidirectional exchange, rwightman_sigmoid_loss.py:75-107) instead of r, r+1, r+2, ...;
                            same pairs, same result up to fp32 summation order. Collective: set on all ranks */
  SIGLIP_OPT_INPUT_F16 = 13, /* 1: the img / txt buffers handed to siglip_forward / siglip_backward / siglip_fwd_bwd hold IEEE
                                fp16 values 16*x (what siglip_convert_f32 and siglip_normalize_fwd then produce) instead of
                                bf16: 11 significant bits for callers with fp32 embeddings (the reference's own test feeds fp32,
                                test_distributed_sigmoid_loss.py:57-68; bf16 rounding of such inputs costs 1.7e-3 in the
                                gradients, this format 2e-4). Same on all ranks. Default 0 */
  SIGLIP_OPT_GRAD_TILE_N = 14, /* 0, 128 or 256; accepted, no effect on sm_90a: every column tile is 128 wide (the wgmma
                                  accumulator lives in registers) */
  SIGLIP_OPT_PEER_TIMEOUT_MS = 15, /* bound of every in-kernel wait on a PEER rank (text-ready / contribution-ready /
                                      buffer-free flags, scalar exchange). Default 600000 (10 min, the order of a process
                                      group's collective timeout: a peer may be late by a checkpoint save or an evaluation
                                      pass); also settable by the environment variable SIGLIP_PEER_TIMEOUT_MS at context
                                      creation. On expiry the kernel records the wait site and traps: the next call
                                      returns SIGLIP_ERR_CUDA naming it. Waits on the kernel's own mbarriers keep their
                                      4 s bound. */
  SIGLIP_OPT_INKERNEL_SYNC = 16, /* 1 (default): siglip_fwd_bwd waits for / raises every cross-rank flag inside its wgmma
                                    kernels (a W-rank step is exactly 2W launches); 0: separate one-block wait / signal
                                    kernels and a copy around them (A/B measurements) */
  SIGLIP_OPT_SPLIT_K = 17, /* gradient kernel, tiles of a ragged last wave: 0 (default) never split; -1 split them
                              floor(units / tiles) ways (at most 4) along K; S = 2..8 at most S ways (fp32 partials
                              through a workspace, fixed-order sum: bitwise independent of which CTA finishes first).
                              Measured: no gain at the shapes tried (the last wave is not what a short launch waits for),
                              so it stays opt-in */
  SIGLIP_OPT_PDL = 19, /* 1 (default): the wgmma kernels are launched with programmatic stream serialization: their
                          set-up (barrier initialisation, descriptor prefetch) overlaps the tail of the previous kernel
                          of the stream; griddepcontrol.wait orders every global access behind it. 0: plain launches */
  SIGLIP_OPT_TPRIME_F64 = 20, /* 1: the t_prime pointer given to siglip_forward / siglip_backward / siglip_fwd_bwd(_scaled)
                                 is an fp64 device scalar — the dtype of the reference's parameter
                                 (torch.tensor(np.log(10)), distributed_sigmoid_loss.py:11) — and dt_prime is written as
                                 fp64: the module hands its parameter over without a conversion kernel. Default 0 (fp32) */
  SIGLIP_OPT_AUX_TRACE = 18 /* 1: record globaltimer stamps of the auxiliary warps of CTA 0 for every launch (start,
                               last peer flag seen, jobs done, end of launch); read with siglip_ctx_aux_trace */
};

/* Library / build identification: "siglip_b200 <version> sm_90a". */
const char* siglip_version(void);

/* Text of the last error on the calling thread ("" if none). */
const char* siglip_last_error(void);

/* Number of CUDA devices with compute capability 9.x visible to the process (0 on a CPU-only box). */
int siglip_device_count(void);

/*
 * Create the per-process context: replaces DDPSigmoidLoss.__init__ (distributed_sigmoid_loss.py:9-15) —
 * `B` is its gpu_batch_size, `rank`/`world` what dist.get_rank()/get_world_size() return at :37-38.
 * Allocates the workspaces (gathered text [world*B, D] bf16, per-owner dtxt slots [world][B, D] fp32, reduction partials,
 * flags); the [Bp, Bp] 16-bit sigma operands and the fp16 text copies that go with them are allocated on first use: two for
 * the fused step whatever the world size, one per rank for the split forward / backward API (an allocation failure there
 * says how many GiB were needed). On any failure nothing stays allocated. `device` is the CUDA device ordinal.
 */
int siglip_ctx_create(siglip_ctx** out, int device, int rank, int world, int B, int D);

/*
 * Same, for ranks with DIFFERENT batch sizes: batch_per_rank[p] is rank p's batch (every rank passes the same list).
 * The reference cannot express this (its labels are gpu_batch_size x gpu_batch_size, distributed_sigmoid_loss.py:26-30,
 * and all_gather needs equal shapes); semantics follow it where defined: rank r's loss sums its B_r images against all
 * sum(B) texts and divides by ITS batch B_r (:47), the text gradient of rank c sums the contributions of every rank.
 */
int siglip_ctx_create_uneven(siglip_ctx** out, int device, int rank, int world, const int* batch_per_rank, int D);

int siglip_ctx_set_option(siglip_ctx* ctx, int option, int value);

/* Bytes of workspace the context holds on the device. */
size_t siglip_ctx_workspace_bytes(const siglip_ctx* ctx);

/*
 * Peer-memory bootstrap (replaces the process-group plumbing the reference gets from
 * dist_nn.all_gather, distributed_sigmoid_loss.py:35, and batch_isend_irecv, distributed_utils.py:24,57):
 * each rank exports CUDA-IPC handles of its text / dtxt-slot / flag buffers; the caller all-gathers the
 * byte strings over any transport (torch.distributed.all_gather_object) and hands the concatenation back.
 * Not needed when world == 1.
 */
size_t siglip_ctx_handle_bytes(void);
int siglip_ctx_export_handles(siglip_ctx* ctx, void* out_bytes, size_t capacity);
int siglip_ctx_import_handles(siglip_ctx* ctx, const void* all_ranks_bytes, size_t bytes_per_rank);

/*
 * One training step of the loss, fused: replaces DDPSigmoidLoss.forward (distributed_sigmoid_loss.py:17-48) AND
 * the autograd backward of it (SURVEY.md §3.2), i.e. loss plus the four gradients for upstream grad 1:
 *   loss      [1]    = (1/B) sum_ij softplus(-y_ij z_ij)
 *   dimg      [B,D]  = dloss/dimg           (this rank's loss only)
 *   dtxt      [B,D]  = d(sum over ranks of their losses)/dtxt   (what all_gather's backward delivers)
 *   dt_prime  [1], dbias [1]                (this rank's loss only; DDP averages them later)
 * Collective: every rank of the context's world must call it the same number of times.
 * Loss and gradient kernels alternate chunk by chunk (L0 L1 G1 L2 G2 ... G0), so only TWO [B, B] sigma operands exist
 * however many ranks there are (the split siglip_forward / siglip_backward keep one per rank between the two calls),
 * and every cross-rank flag is waited for / raised inside the kernels: a W-rank step is exactly 2W launches.
 * A single-rank step performs no host synchronisation and no allocation after the first call and can be captured into a
 * CUDA graph; a multi-rank step cannot (its flag values advance every step) and returns SIGLIP_ERR_STATE under capture.
 */
int siglip_fwd_bwd(siglip_ctx* ctx, const void* img, const void* txt, const float* t_prime, const float* bias,
                   float* loss, void* dimg, void* dtxt, float* dt_prime, float* dbias, void* cuda_stream);
/* Same with an upstream gradient: every gradient is multiplied by *grad_out (device scalar; NULL = 1) in the kernel
 * epilogues (autograd's grad_output of the loss, known before the step when the loss is the last node of the graph). */
int siglip_fwd_bwd_scaled(siglip_ctx* ctx, const void* img, const void* txt, const float* t_prime, const float* bias,
                          const float* grad_out, float* loss, void* dimg, void* dtxt, float* dt_prime, float* dbias,
                          void* cuda_stream);

/*
 * L2 normalisation fused around the loss (the step the reference's callers run immediately before it:
 * F.normalize, test_distributed_sigmoid_loss.py:99-101, README.md:34). [B, D] rows, D % 8 == 0:
 *   fwd: xhat = bf16(x / max(||x||, 1e-12)) (fp16(16 xhat) under SIGLIP_OPT_INPUT_F16) and inv_norm[r] = 1 / max(||x_r||, 1e-12); x is fp32 (in_bf16 = 0) or bf16
 *   bwd: dx = inv_norm * (dxhat - xhat <xhat, dxhat>) with xhat recomputed in fp32 from x; dxhat fp32 or bf16
 *        (grad_bf16), dx in x's dtype — autograd's backward of F.normalize composed with the loss gradients.
 */
int siglip_normalize_fwd(siglip_ctx* ctx, const void* x, int in_bf16, void* xhat_bf16, float* inv_norm,
                         void* cuda_stream);
/* [B, D] fp32 -> the 16-bit operand format the context currently expects (bf16, or fp16(16 x) under
 * SIGLIP_OPT_INPUT_F16): the cast the module applies to fp32 embeddings (replaces `.to(bfloat16)`). */
int siglip_convert_f32(siglip_ctx* ctx, const float* x_f32, void* out_16bit, void* cuda_stream);
int siglip_normalize_bwd(siglip_ctx* ctx, const void* x, int in_bf16, const float* inv_norm, const void* dxhat,
                         int grad_bf16, void* dx, void* cuda_stream);

/*
 * dst = src * (*g) elementwise over `nbytes` (any whole number of elements) of fp32 (is_bf16 = 0) or bf16 (is_bf16 = 1) data: the whole
 * `backward()` of the module — the fused step already produced the gradients for an upstream gradient of 1
 * (replaces the autograd graph replay of SURVEY.md §3.2). `g` is a device scalar (grad_output).
 */
int siglip_scale(siglip_ctx* ctx, const void* src, void* dst, size_t nbytes, int is_bf16, const float* g,
                 void* cuda_stream);

/*
 * The same step as two calls, the shape autograd wants:
 *   siglip_forward  — the W loss kernels; with save_for_backward != 0 it also keeps, inside the context, the sigma
 *                     operands, the fp16 operand copies and dt'/dbias that the backward needs (replaces the autograd
 *                     graph the reference records at distributed_sigmoid_loss.py:22-33);
 *   siglip_backward — the W gradient kernels on that saved state, every gradient multiplied by the upstream scalar
 *                     `grad_out` (device pointer; NULL = 1) in the kernel epilogue (replaces the graph replay,
 *                     SURVEY.md §3.2). `img` / `txt` must be the buffers given to the forward.
 * Both are collectives over the context's world. siglip_ctx_saved_generation() identifies the saved state (0 = none):
 * a backward must follow the forward that produced the generation it expects (the Python mirror re-runs the forward if
 * another forward intervened).
 */
int siglip_forward(siglip_ctx* ctx, const void* img, const void* txt, const float* t_prime, const float* bias,
                   float* loss, int save_for_backward, void* cuda_stream);
int siglip_backward(siglip_ctx* ctx, const void* img, const void* txt, const float* t_prime, const float* grad_out,
                    void* dimg, void* dtxt, float* dt_prime, float* dbias, void* cuda_stream);
unsigned long long siglip_ctx_saved_generation(const siglip_ctx* ctx);

/* Forward only (torch.no_grad / evaluation): siglip_forward with save_for_backward = 0. */
int siglip_fwd(siglip_ctx* ctx, const void* img, const void* txt, const float* t_prime, const float* bias,
               float* loss, void* cuda_stream);

/*
 * Same step with HOST buffers (pinned or pageable): host->device copies of img/txt, the step, and
 * device->host copies of loss (+ gradients when the pointers are non-null) all inside the call, which returns
 * after the step has finished (= siglip_host_submit + siglip_host_wait). fp32 gradients stay in device staging
 * unless dimg_host / dtxt_host are given.
 *
 * siglip_host_submit / siglip_host_wait: the same end-to-end step, pipelined. submit enqueues the host->device copies
 * of THIS step's inputs on an internal copy stream (two staging sets), the step on cuda_stream behind them and the
 * device->host copy of (loss, dt_prime, dbias) behind that, and returns a ticket; wait blocks until that step's
 * results are on the host. At most two steps may be in flight: submit blocks on the step that used the same staging
 * set. The copies of step n+1 overlap the kernels of step n; every step still pays its own copies.
 * This is the end-to-end entry the benchmark times. Host buffers must stay valid until the step's wait returns.
 */
int siglip_host_submit(siglip_ctx* ctx, const void* img_host, const void* txt_host, float t_prime, float bias,
                       unsigned long long* ticket, void* cuda_stream);
/* Same, and the step's dimg / dtxt also travel back: bf16 [B, D] each into the given host buffers (both or neither),
 * copied on a second internal copy stream so that the read-back of step n overlaps the kernels of step n+1. */
int siglip_host_submit_grads(siglip_ctx* ctx, const void* img_host, const void* txt_host, float t_prime, float bias,
                             void* dimg_host_bf16, void* dtxt_host_bf16, unsigned long long* ticket,
                             void* cuda_stream);
int siglip_host_wait(siglip_ctx* ctx, unsigned long long ticket, float* loss_host, float* dt_prime_host,
                     float* dbias_host);
int siglip_fwd_bwd_host(siglip_ctx* ctx, const void* img_host, const void* txt_host, float t_prime, float bias,
                        float* loss_host, float* dimg_host, float* dtxt_host, float* dt_prime_host,
                        float* dbias_host, void* cuda_stream);

/*
 * With SIGLIP_OPT_KERNEL_TIMING on: device-synchronise, then return the summed CUDA-event durations (ms) and the
 * launch counts of the loss kernel and of the gradient kernel since the previous call (for the roofline line
 * of the benchmark). Resets the accumulation.
 */
int siglip_ctx_kernel_times(siglip_ctx* ctx, double* loss_ms, int* loss_launches, double* grad_ms,
                            int* grad_launches);

/* Kernels launched by the context since creation (for the benchmark's gpu_launches field). */
unsigned long long siglip_ctx_launch_count(const siglip_ctx* ctx);

/*
 * Test hook: plain contraction C[M,N] (fp32) = A * B^T on the same wgmma mainloop, to pin the operand
 * layouts independently of the loss epilogue. a_mn / b_mn: 0 = operand stored [rows][K] (K contiguous),
 * 1 = stored [K][rows] (rows contiguous). lda/ldb/ldc in elements. cta_group 1 or 2.
 */
int siglip_debug_gemm(int device, int cta_group, int M, int N, int K, const void* A, long long lda, int a_mn,
                      const void* Bm, long long ldb, int b_mn, float* C, long long ldc, void* cuda_stream);

/* Same contraction launched `iters` times back to back (after one warm-up when iters > 1); *ms_per_iter receives
 * the CUDA-event time per launch. Used to tune the mainloop apart from the loss epilogue. */
int siglip_debug_gemm_timed(int device, int cta_group, int M, int N, int K, const void* A, long long lda, int a_mn,
                            const void* Bm, long long ldb, int b_mn, float* C, long long ldc, int iters,
                            float* ms_per_iter, void* cuda_stream);

/*
 * Test hooks for exercising the multi-chunk schedule of ONE rank on ONE GPU (world > 1 context, no peers):
 * loopback wires every "peer" pointer to the context's own buffers (the peers' contribution slots to a zero buffer);
 * the test preloads the text chunks of the other ranks, runs the step, and reads this rank's per-owner dtxt
 * contributions back: slot c for c != rank, and the dtxt OUTPUT of the step for the own chunk (own contribution + the
 * zero "peer" contributions).
 */
int siglip_debug_loopback(siglip_ctx* ctx);
int siglip_debug_set_text_chunk(siglip_ctx* ctx, int chunk, const void* txt_dev, void* cuda_stream);
int siglip_debug_get_slot(siglip_ctx* ctx, int chunk, float* out_dev, void* cuda_stream);
/* Loopback only: seed the (dt_prime, dbias) mailbox standing in for peer rank `peer`, so that the mean computed under
 * SIGLIP_OPT_SYNC_SCALAR_GRADS can be checked against numbers the kernel did not produce itself. */
int siglip_debug_set_mailbox(siglip_ctx* ctx, int peer, float dt_prime, float dbias);
/* With SIGLIP_OPT_AUX_TRACE: device-synchronise and copy out 16 globaltimer stamps (ns) per launch since the last call:
 * [0..2] auxiliary warps of CTA 0: start, last peer flag observed (0 = no wait), jobs done; [3] launch end as seen by
 * the last CTA; [4] kernel entry (CTA 0); [5] set-up done (barriers); [6] MMAs of the first tile done (CTA 0);
 * [7] last tile done (CTA 0); [8] first CTA finished; [9] / [10] latest / earliest "last tile done" over the CTAs;
 * [11] last CTA through the epilogue of its tiles; [12] / [13] last / first CTA to enter the kernel; [14] last CTA through
 * its set-up; [15] unused. `out` holds 16 * max_launches values. */
int siglip_ctx_aux_trace(siglip_ctx* ctx, unsigned long long* out, int max_launches, int* n_launches);

void siglip_ctx_destroy(siglip_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* SIGLIP_B200_H_ */
