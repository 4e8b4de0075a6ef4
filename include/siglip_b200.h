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
 * Data layout: `img` is a row-major [R, D] bf16 device buffer (R = B unless the context was created with
 * siglip_ctx_create_extras: then this rank's R images are its B paired images followed by its extra images), `txt` a
 * row-major [T, D] one (T = B unless the context was created with siglip_ctx_create_texts / _extras: then this rank's T
 * texts are its B paired captions followed by its hard negatives), 16-byte aligned, D % 8 == 0. `dimg` [R, D] and
 * `dtxt` [T, D] are row-major fp32 (or bf16 with SIGLIP_OPT_GRAD_BF16). Scalars are fp32 device scalars.
 * Non-finite inputs: NaN and +-inf embedding entries, t' and bias reach every output they touch (every conversion to an
 * operand format keeps them), so each output element is non-finite where float64 autograd of the loss on the same
 * operand values is (NaN and inf are not told apart), and per-sample losses are NaN or +inf as documented there.
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
 *   SIGLIP_DEBUG_MCAST, _AB_F16, _AB_FP8, _WAITSTATS, _STAGES, _TILE_N (128 or 256)   variants of
 *                                siglip_debug_gemm(_timed) only
 */

/* tuning knobs (siglip_ctx_set_option) */
enum {
  SIGLIP_OPT_CTA_GROUP = 1, /* 1: every CTA computes its own 128-row tile; 2 (default): clusters of two CTAs on adjacent
                               128-row blocks share the B tile by TMA multicast. Loss-kernel tiles are 128 columns
                               wide, gradient-kernel tiles 128 or 256 (SIGLIP_OPT_GRAD_TILE_N) */
  SIGLIP_OPT_OVERLAP_PULL = 2, /* 1 (default): pull the next text chunk inside the loss kernel; 0: separate copy */
  SIGLIP_OPT_KERNEL_TIMING = 3, /* 1: bracket every loss / gradient kernel launch with CUDA events on the caller's stream */
  SIGLIP_OPT_STAGES_LOSS = 4,  /* TMA->MMA pipeline depth of the loss kernel: 0 (default, = 6), 4 or 6 */
  SIGLIP_OPT_STAGES_GRAD = 5,  /* ... of the gradient kernel with 128-column tiles; 256-column tiles (48 KiB per stage)
                                  always run 4 stages, whatever is asked */
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
  SIGLIP_OPT_GRAD_TILE_N = 14, /* column tiles of the gradient kernel: 128 (wgmma m64n128), 256 (m64n256: one
                                  instruction per k step instead of two, a third less operand traffic per FLOP) or 0
                                  (default): 256 when 1.8 x its waves over the persistent grid are at most the waves
                                  of 128-column tiles (B = 16384 with D = 768, 1024 or 1152), else 128 (D <= 128,
                                  B = 16384 with D = 384, B = 4096 with D = 768). Same results bit for bit. Split-K
                                  (SIGLIP_OPT_SPLIT_K with SIGLIP_OPT_MCAST 1) always takes 128 */
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
  SIGLIP_OPT_SAMPLE_IDS = 21, /* 1: labels from per-sample ids instead of positions. Image i of rank r and text j of rank c
                                 are a positive pair iff ids_r[i] == ids_c[j] (repeated captions, several captions per
                                 image, a sample drawn on two ranks); loss and gradients keep their formulas with these
                                 labels. Every step takes this rank's ids from siglip_set_sample_ids; the ids travel to the
                                 other ranks with the text. Unique ids give exactly the default labels (and bit-identical
                                 results). Off-diagonal positives enter the gradient contractions through the fp16 sigma
                                 operand (2^-12 relative rounding each, like the negatives). The host-buffer entries are
                                 unavailable in this mode. Collective: set on all ranks. Default 0 */
  SIGLIP_OPT_EXTRA_TEXT_IDS = 22, /* 1: the extra texts of a siglip_ctx_create_texts context carry ids too (several
                                     captions per image). Text j of chunk c has id text_ids_c[j]: sample_ids_c[j] for
                                     j < B_c, and the extra's own id (siglip_set_extra_text_ids) for j >= B_c. Pair (i, j)
                                     is positive iff sample_ids_r[i] == text_ids_c[j], on any rank: an extra that carries
                                     an image's id is another caption of that image, an extra whose id matches no image
                                     is a hard negative. The loss still divides by the image batch B_r. Needs
                                     SIGLIP_OPT_SAMPLE_IDS on (else SIGLIP_ERR_STATE); turning that option off clears this
                                     one. Accepted on any context; with T == B it changes nothing. Collective: set on all
                                     ranks. Default 0 */
  SIGLIP_OPT_SAMPLE_WEIGHTS = 23, /* 1: per-sample loss weights. Rank r's images carry weights a_r[i], the texts of
                                     chunk c (paired, then extras) weights c_c[j], all in [0, 1]; pair (i, j) has weight
                                     w_ij = a_r[i] c_c[j] and rank r's loss is (1/B_r) sum_ij w_ij softplus(-y_ij z_ij)
                                     (labels as without weights), with every gradient following (G_ij = w_ij x the
                                     unweighted term). Still divided by B_r. A sample whose image and text weights are
                                     both 0 leaves loss and gradients exactly, at the same shapes; unit weights give
                                     bit-identical results. Every step takes this rank's weights from
                                     siglip_set_sample_weights; the text weights travel to the other ranks with the text.
                                     Retrieval metrics ignore the weights. The host-buffer entries are unavailable in
                                     this mode. Collective: set on all ranks. Default 0 */
  SIGLIP_OPT_EXTRA_IMAGE_IDS = 24, /* 1: the extra images of a siglip_ctx_create_extras context carry ids too (several
                                      images per caption). Image i of rank r has id row_ids_r[i]: sample_ids_r[i] for
                                      i < B_r, the extra's own id (siglip_set_extra_image_ids) for i >= B_r. Pair (i, j)
                                      is positive iff row_ids_r[i] == text_ids_c[j], on any rank: an extra image with a
                                      caption's id is another image of that caption, one whose id matches no text is a
                                      hard-negative image. Without this option an extra image matches no id. The loss
                                      still divides by B_r. Needs SIGLIP_OPT_SAMPLE_IDS on (else SIGLIP_ERR_STATE);
                                      turning that option off clears this one. Collective: set on all ranks. Default 0 */
  SIGLIP_OPT_DISTILL = 25, /* 1: distillation from a frozen teacher (siglip_ctx_create_distill and
                              siglip_ctx_create_distill_extras contexts only, else SIGLIP_ERR_STATE). The target of pair (i, j) becomes
                                q_ij = (1 - lambda) y_ij + lambda sigma(t_T <timg_i, ttxt_j> + b_T)
                              (y in {0, 1}: the labels the other options give; 0 for a hard negative) and rank r's
                              loss
                                (1/B_r) sum_ij w_ij (softplus(z_ij) - q_ij z_ij).
                              An extra text or image takes its teacher probability from its own teacher row. An
                              excluded pair (SIGLIP_OPT_EXCLUDE_GROUPS) adds exactly 0. The teacher similarities are
                              computed tile by tile inside the loss kernel and never stored; the teacher texts travel
                              with the student texts. Every step needs siglip_set_teacher since the previous step (else
                              SIGLIP_ERR_STATE before any launch). Composes with ids, weights, metrics, row panels,
                              bidir and uneven batches. On a siglip_ctx_create_distill_extras context it also composes
                              with extras, excluded groups, label sets, per-sample losses and top-K; a
                              siglip_ctx_create_distill context refuses those (SIGLIP_ERR_STATE). Never with
                              SIGLIP_OPT_FOCAL, nor in the host-buffer entries. Per-sample losses sum the terms w_ij (softplus(z_ij) - q_ij z_ij) >= 0; metrics
                              and top-K rank the student's logits. The gradient kernels are unchanged. Collective.
                              Default 0 */
  SIGLIP_OPT_SIGMA_BUDGET_MIB = 26, /* bound, in MiB, of the 16-bit sigma operands (the one buffer that grows with B^2).
                                       0 (default): none, every step as before. Otherwise siglip_fwd_bwd scores the
                                       rank's R rows in row panels of P rows, P the largest multiple of
                                       128 x cluster_size (SIGLIP_OPT_CTA_GROUP x SIGLIP_OPT_MCAST) whose buffers fit:
                                       2 buffers of [P, Tp] at W > 1, 1 at W = 1 (siglip_sigma_panel_rows). A budget that
                                       holds the whole operands runs the unbounded step unchanged; one below a minimal
                                       panel is refused (SIGLIP_ERR_INVALID, with the minimum). P depends on the budget,
                                       the shapes and the cluster options, never on free memory. Composes with every
                                       other option. Retrieval metrics and per-sample losses are bit-identical to the
                                       unbounded step, and so is dimg at W = 1 without split-K. At W > 1 the dimg rows
                                       of panels past 0 add the own chunk's term first rather than last, and split-K
                                       slices a panel's ragged wave differently: dimg then agrees up to fp32 summation
                                       order, as loss / dtxt / dt' / dbias always do (DESIGN.md, "Row panels"). siglip_fwd / siglip_forward without save allocate one
                                       panel at most; siglip_forward with save keeps W whole operands until the backward
                                       and returns SIGLIP_ERR_STATE when they exceed the budget. The host-buffer entries
                                       run siglip_fwd_bwd and so run under the budget. Setting it releases the operands
                                       (and any forward saved for backward). Per rank; default 0 */
  SIGLIP_OPT_EXCLUDE_GROUPS = 27, /* 1: pairs of the same group are excluded from the loss. Every image (paired, then
                                     extra: [R_r]) and every text (paired, then extra: [T_r]) carries an int64 group id;
                                     a negative id is "no group". A pair that the other options make positive stays
                                     positive; any other pair (i, j) with image_group[i] == text_group[j] >= 0 adds
                                     exactly 0 to the loss, the sigma operand, dt' / dbias, dimg / dtxt and the
                                     per-sample losses (the loss still divides by B_r). Metrics and top-K lists are
                                     unchanged. Every step needs siglip_set_groups since the previous step (else
                                     SIGLIP_ERR_STATE before any launch); the text groups travel to the other ranks with
                                     the text. Unavailable with SIGLIP_OPT_DISTILL on a siglip_ctx_create_distill
                                     context, and in the host-buffer entries (SIGLIP_ERR_STATE). Collective.
                                     Default 0 */
  SIGLIP_OPT_LABEL_SETS = 28, /* 1: multi-label positives (siglip_ctx_create_labels contexts and
                                 siglip_ctx_create_distill_extras contexts with M > 0 only, else SIGLIP_ERR_STATE). Every sample carries a set of M int64 labels (a negative entry is an
                                 empty slot; duplicates are allowed), shared by its image and its paired text; extra
                                 texts and extra images carry their own. Pair (image i, text j) is positive iff it is the
                                 own-chunk positional pair (i == j < B_r on the own chunk) or the two sets share a label
                                 >= 0; every other pair is negative. Loss and gradients keep their formulas (the loss
                                 divides by B_r); the own diagonal keeps its fp32 term, other positives go through the
                                 sigma operand like id positives. M = 1 with labels >= 0 is SIGLIP_OPT_SAMPLE_IDS with
                                 those ids (under ids, -1 is an ordinary id; here it is an empty slot). Excluded groups
                                 apply after these positives. Metrics and top-K lists count a hit by the same rule and
                                 rank all R_r images (i2t) and all T_r texts (t2i). Every step needs siglip_set_label_sets
                                 since the previous step (else SIGLIP_ERR_STATE before any launch); the text sets travel
                                 to the other ranks with the text. Unavailable with SIGLIP_OPT_SAMPLE_IDS,
                                 SIGLIP_OPT_EXTRA_TEXT_IDS, SIGLIP_OPT_EXTRA_IMAGE_IDS and in the host-buffer entries
                                 (SIGLIP_ERR_STATE). Collective. Default 0 */
  SIGLIP_OPT_FOCAL = 29, /* 1: the focal pair loss (torchvision's sigmoid_focal_loss) in place of the SigLIP term. Pair
                            (i, j) with target y (from whatever labels the other options give), p = sigma(z),
                            p_t = y ? p : 1 - p and a_t = y ? alpha : 1 - alpha (1 without alpha) adds
                            w a_t (1 - p_t)^gamma softplus(-(2y - 1) z) to the loss (still divided by B_r), and the
                            gradients, dt' and dbias follow. gamma = 0 without alpha is the SigLIP loss. Excluded pairs
                            stay 0; metrics and top-K lists are unchanged; per-sample losses sum the focal terms. gamma
                            and alpha come from siglip_set_focal: a step in the mode before that call returns
                            SIGLIP_ERR_STATE before any launch. Unavailable with SIGLIP_OPT_DISTILL and in the
                            host-buffer entries (SIGLIP_ERR_STATE). Collective: every rank sets the same option and
                            values (not checked). Default 0 */
  SIGLIP_OPT_AUX_TRACE = 18 /* 1: record globaltimer stamps of the auxiliary warps of CTA 0 for every launch (start,
                               last peer flag seen, jobs done, end of launch); read with siglip_ctx_aux_trace */
};

/*
 * Panel height of SIGLIP_OPT_SIGMA_BUDGET_MIB, without a device: `rows` (R) rows of a rank, sigma operands of
 * `rows_padded` x `cols_padded` (Rp x Tp, max R and max T rounded up to 256) 16-bit elements, `buffers` of them (2 at
 * W > 1, 1 at W = 1), panels a multiple of `cluster_rows` (128 x cluster size). Returns the panel height: `rows` when one
 * panel covers the rank (budget 0, or one that holds the whole operands), 0 when the budget is below one minimal panel,
 * -SIGLIP_ERR_INVALID for invalid arguments. *buffer_rows (optional) receives the rows of each allocated operand.
 */
int siglip_sigma_panel_rows(int rows, int rows_padded, int cols_padded, int buffers, int cluster_rows, int budget_mib,
                            int* buffer_rows);

/*
 * The same rule for a context's shapes, cluster options and budget: `buffers` sigma operands (0: what siglip_fwd_bwd
 * keeps, 2 at W > 1 and 1 at W = 1; the world size: what siglip_forward with save keeps). *panel_rows gets the panel
 * height (0: below one minimal panel), *panels the number of panels, *whole 1 when the budget holds the whole operands
 * (the unbounded layout). Any output may be null. Host only.
 */
int siglip_ctx_sigma_panels(const siglip_ctx* c, int buffers, int* panel_rows, int* panels, int* whole);

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
 * The first sigma operand is allocated at creation when the device holds it; when it runs out of memory for it, the
 * context is created all the same and the first step allocates what it needs (under SIGLIP_OPT_SIGMA_BUDGET_MIB: one
 * panel's worth) or reports the shortfall.
 */
int siglip_ctx_create(siglip_ctx** out, int device, int rank, int world, int B, int D);

/*
 * Same, for ranks with DIFFERENT batch sizes: batch_per_rank[p] is rank p's batch (every rank passes the same list).
 * The reference cannot express this (its labels are gpu_batch_size x gpu_batch_size, distributed_sigmoid_loss.py:26-30,
 * and all_gather needs equal shapes); semantics follow it where defined: rank r's loss sums its B_r images against all
 * sum(B) texts and divides by ITS batch B_r (:47), the text gradient of rank c sums the contributions of every rank.
 */
int siglip_ctx_create_uneven(siglip_ctx** out, int device, int rank, int world, const int* batch_per_rank, int D);

/*
 * Same, with HARD-NEGATIVE captions (NegCLIP-style / compositionality fine-tuning: perturbed captions that belong to
 * no image). Rank p holds images_per_rank[p] = B_p images and texts_per_rank[p] = T_p >= B_p texts: texts 0 .. B_p - 1
 * are the captions of its images, texts B_p .. T_p - 1 its K_p = T_p - B_p hard negatives. The global text batch is the
 * concatenation over ranks of [paired, extras] (global text index = prefix sum of T + local index). Rank r's loss is
 *   (1/B_r) sum_i sum_{j over all sum(T) texts} softplus(-y_ij z_ij)
 * with y = +1 for the positional pair (or, under SIGLIP_OPT_SAMPLE_IDS, a PAIRED text with the same id) and -1 for
 * everything else: an extra is never positive, whatever the ids. txt / dtxt of every step are [T_r, D] (dtxt includes
 * the extras' rows: the gradient of the sum over ranks of their losses); dt' / dbias include the extras' terms. Sample
 * ids stay [B_r] (they describe the paired texts); SIGLIP_OPT_EXTRA_TEXT_IDS gives the extras ids of their own, so that
 * they can be further captions of an image. The host-buffer entries are unavailable (SIGLIP_ERR_STATE).
 * Workspaces: the text-shaped ones (gathered text, dtxt slots, fp16 text copies) hold max(T) rows per chunk and the
 * sigma operands are [Bp, Tp] (max B, max T rounded up to 256). Time grows with T / B like the FLOPs (6 B T D).
 * Every rank passes the same two lists; texts_per_rank == images_per_rank is exactly siglip_ctx_create_uneven.
 * Invalid arguments return SIGLIP_ERR_INVALID before any device work.
 */
int siglip_ctx_create_texts(siglip_ctx** out, int device, int rank, int world, const int* images_per_rank,
                            const int* texts_per_rank, int D);

/*
 * Same, with EXTRA IMAGES as well (several images per caption: product photos, video frames, augmented crops; or
 * hard-negative images). Rank p has batch_per_rank[p] = B_p paired samples, images_per_rank[p] = R_p >= B_p images and
 * texts_per_rank[p] = T_p >= B_p texts: images 0 .. B_p - 1 are paired with texts 0 .. B_p - 1, images B_p .. R_p - 1
 * are its E_p = R_p - B_p extra images. Rank r's loss is
 *   (1/B_r) sum_{i < R_r} sum_{j over all sum(T) texts} softplus(-y_ij z_ij)
 * (the divisor stays the paired batch). The positional positive is row == col < B_r of the own chunk: an extra image is
 * never a positional positive, and under SIGLIP_OPT_SAMPLE_IDS it matches no id unless SIGLIP_OPT_EXTRA_IMAGE_IDS gives
 * it one. img / dimg of every step are [R_r, D]; dtxt contracts over all R_r rows of every rank; dt' / dbias include
 * the extras' terms. Images never leave their rank: the text exchange is unchanged, and the only new cross-rank data are
 * the extra images' ids of a metrics step. Workspaces: the sigma operands are [Rp, Tp] (max R rounded up to 256), the
 * fp16 image copy and the running dimg hold R rows. Time grows with R / B like the FLOPs (6 R T D). With
 * images_per_rank == batch_per_rank this is exactly siglip_ctx_create_texts. Every rank passes the same three lists.
 * The host-buffer entries are unavailable (SIGLIP_ERR_STATE). Invalid arguments return SIGLIP_ERR_INVALID before any
 * device work.
 */
int siglip_ctx_create_extras(siglip_ctx** out, int device, int rank, int world, const int* batch_per_rank,
                             const int* images_per_rank, const int* texts_per_rank, int D);

/*
 * Same as siglip_ctx_create_uneven, for distillation (SIGLIP_OPT_DISTILL): D_teacher is the width of the teacher's
 * embeddings (a positive multiple of 8; it may differ from D). The gathered teacher text ([world][max B, D_teacher]
 * bf16 or fp16 x 16) is part of the exported text allocation, sized here because options are set after the handle
 * exchange; every rank passes the same list and D_teacher (handle import refuses a peer whose D_teacher differs).
 * D_teacher = 0 is exactly siglip_ctx_create_uneven.
 */
int siglip_ctx_create_distill(siglip_ctx** out, int device, int rank, int world, const int* batch_per_rank, int D,
                              int D_teacher);

/* Labels per set at most (siglip_ctx_create_labels) */
#define SIGLIP_MAX_LABELS 4

/*
 * Same as siglip_ctx_create_extras, for label sets (SIGLIP_OPT_LABEL_SETS): every sample, extra text and extra image
 * carries a set of M labels, 1 <= M <= SIGLIP_MAX_LABELS. The gathered text sets ([world][T_max, M] int64, followed by
 * the text groups) are part of the exported text allocation, sized here because options are set after the handle
 * exchange; every rank passes the same lists and M (handle import refuses a peer whose M differs). A context created
 * any other way keeps its layout, and SIGLIP_OPT_LABEL_SETS returns SIGLIP_ERR_STATE there.
 */
int siglip_ctx_create_labels(siglip_ctx** out, int device, int rank, int world, const int* batch_per_rank,
                             const int* images_per_rank, const int* texts_per_rank, int D, int M);

/*
 * A context that holds everything at once: a teacher of width D_teacher (a positive multiple of 8, as in
 * siglip_ctx_create_distill), extra texts and extra images (as in siglip_ctx_create_extras) and, for M in
 * 1 .. SIGLIP_MAX_LABELS, label sets (as in siglip_ctx_create_labels; M = 0: none). The gathered teacher text is
 * [world][T_max, D_teacher]: every text of a rank, paired then extras, has a teacher row. Handle import refuses a peer
 * whose D_teacher or M differs. Under SIGLIP_OPT_DISTILL such a context takes per-sample losses, top-K, excluded
 * groups and label sets, which a siglip_ctx_create_distill context refuses. siglip_ctx_create_distill has the layout
 * of this entry with images = texts = batch and M = 0, and siglip_ctx_create_labels that of this entry without a
 * teacher.
 */
int siglip_ctx_create_distill_extras(siglip_ctx** out, int device, int rank, int world, const int* batch_per_rank,
                                     const int* images_per_rank, const int* texts_per_rank, int D, int D_teacher,
                                     int M);

/*
 * SIGLIP_OPT_DISTILL: the teacher of the NEXT step. timg [R, D_teacher] and ttxt [T, D_teacher] are this rank's teacher
 * embeddings in the order of the student's (paired rows, then extras; R = T = B without extras), both bf16 (teacher_f16 = 0) or both fp16(x * 16) (teacher_f16 = 1, the fp32-input format), 16-byte
 * aligned; t_prime_T / bias_T are fp32 device scalars (t_T = exp(t_prime_T)); lambda in (0, 1]. Only the pointers are
 * recorded (like siglip_request_metrics): the buffers must hold their values when the step runs on its stream, and a
 * single-rank step stays capturable into a CUDA graph. No gradient flows to the teacher.
 */
int siglip_set_teacher(siglip_ctx* ctx, const void* timg, const void* ttxt, int teacher_f16, const float* t_prime_T,
                       const float* bias_T, float lambda);

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
 *   dimg      [B,D]  = dloss/dimg           (this rank's loss only; [R, D] with extra images)
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
/* The three above for `rows` rows instead of B (rows >= 1): e.g. a [T, D] text tensor with hard negatives. */
int siglip_normalize_fwd_rows(siglip_ctx* ctx, int rows, const void* x, int in_bf16, void* xhat_bf16, float* inv_norm,
                              void* cuda_stream);
int siglip_convert_f32_rows(siglip_ctx* ctx, int rows, const float* x_f32, void* out_16bit, void* cuda_stream);
int siglip_normalize_bwd_rows(siglip_ctx* ctx, int rows, const void* x, int in_bf16, const float* inv_norm,
                              const void* dxhat, int grad_bf16, void* dx, void* cuda_stream);

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

/*
 * SIGLIP_OPT_SAMPLE_IDS: the ids of this rank's B samples (image i and text i share ids_dev[i]; int64 device buffer,
 * any values) for the NEXT siglip_fwd_bwd(_scaled) / siglip_forward / siglip_fwd call. They are copied on the stream
 * into the context, so the caller's buffer may be reused once the copy has run; nothing is read on the host (a
 * single-rank step with ids can be captured into a CUDA graph, the copy with it). In ids mode a step without ids set
 * since the previous step returns SIGLIP_ERR_STATE before launching anything; outside it this call returns
 * SIGLIP_ERR_STATE. siglip_backward needs no ids (the saved sigma operand holds the labels).
 */
int siglip_set_sample_ids(siglip_ctx* ctx, const int64_t* ids_dev, void* cuda_stream);

/*
 * SIGLIP_OPT_EXTRA_TEXT_IDS: the ids of this rank's K_r = T_r - B_r extra texts (int64 device buffer of K_r values; may
 * be NULL when K_r = 0) for
 * the NEXT step, copied on the stream like the sample ids (a single-rank step with both copies can be captured into a
 * CUDA graph). In this mode a step needs both this call and siglip_set_sample_ids since the previous step, else it
 * returns SIGLIP_ERR_STATE before launching anything; outside the mode this call returns SIGLIP_ERR_STATE.
 */
int siglip_set_extra_text_ids(siglip_ctx* ctx, const int64_t* ids_dev, void* cuda_stream);

/*
 * SIGLIP_OPT_EXTRA_IMAGE_IDS: the ids of this rank's E_r = R_r - B_r extra images (int64 device buffer of E_r values;
 * may be NULL when E_r = 0) for the NEXT step, copied on the stream into a private [R] row-id buffer behind the sample ids
 * (never exported; a single-rank step with these ids can be captured into a CUDA graph). In this mode a step needs this
 * call and siglip_set_sample_ids since the previous step, else it returns SIGLIP_ERR_STATE before launching anything;
 * outside the mode this call returns SIGLIP_ERR_STATE.
 */
int siglip_set_extra_image_ids(siglip_ctx* ctx, const int64_t* ids_dev, void* cuda_stream);

/*
 * SIGLIP_OPT_SAMPLE_WEIGHTS: this rank's image weights (image_w, [R_r] fp32 device buffer: its paired images, then its
 * extra images; or NULL = ones) and text
 * weights (text_w, [T_r] fp32: its paired texts, then its extras; NULL = ones) for the NEXT siglip_fwd_bwd(_scaled) /
 * siglip_forward / siglip_fwd call. A stream-ordered copy into the context that clamps every value into [0, 1] and maps
 * NaN to 0 (one small kernel launch); nothing is read on the host, so the caller's buffers may be reused once the copy has
 * run and a single-rank step with weights can be captured into a CUDA graph. The first call allocates the context's
 * weight buffer ((round_up(T_r, 4) + R_r) floats; also allowed inside a capture). In the mode a step without this call
 * since the previous step returns SIGLIP_ERR_STATE before launching anything; outside it this call returns
 * SIGLIP_ERR_STATE. siglip_backward needs no weights (the saved sigma operand and positive-pair terms carry them).
 * Weights above 1 do not fit the fp16 sigma operand's range: divide by their maximum and scale the loss by it.
 */
int siglip_set_sample_weights(siglip_ctx* ctx, const float* image_w, const float* text_w, void* cuda_stream);

/*
 * SIGLIP_OPT_EXCLUDE_GROUPS: the group ids of this rank's images (image_groups, [R_r] int64 device buffer: its paired
 * images, then its extra images) and texts (text_groups, [T_r]: its paired texts, then its extras) for the NEXT
 * siglip_fwd_bwd(_scaled) / siglip_forward / siglip_fwd call. Stream-ordered copies into the context: nothing is read on
 * the host, and a single-rank step with groups can be captured into a CUDA graph, the copies with it. In the mode a step
 * without this call since the previous step returns SIGLIP_ERR_STATE before launching anything; outside it this call
 * returns SIGLIP_ERR_STATE.
 */
int siglip_set_groups(siglip_ctx* ctx, const int64_t* image_groups, const int64_t* text_groups, void* cuda_stream);

/*
 * SIGLIP_OPT_LABEL_SETS: the label sets of this rank for the NEXT siglip_fwd_bwd(_scaled) / siglip_forward / siglip_fwd
 * call, int64 device buffers, M labels per row: sample_labels [B, M] (image i and paired text i), extra_text_labels
 * [T - B, M] or NULL (empty sets: pure hard negatives) and extra_image_labels [R - B, M] or NULL (empty sets).
 * Stream-ordered copies into the context: nothing is read on the host, and a single-rank step with label sets can be
 * captured into a CUDA graph, the copies with it. In the mode a step without this call since the previous step returns
 * SIGLIP_ERR_STATE before launching anything; outside it this call returns SIGLIP_ERR_STATE.
 */
int siglip_set_label_sets(siglip_ctx* ctx, const int64_t* sample_labels, const int64_t* extra_text_labels,
                          const int64_t* extra_image_labels, void* cuda_stream);

/*
 * SIGLIP_OPT_FOCAL: gamma (finite, 0 <= gamma <= 8) and alpha (0 <= alpha <= 1, or < 0 for none) of the focal pair loss.
 * Checks and records the two values on the host, launches nothing (a single-rank step stays capturable into a CUDA
 * graph), and they hold for every later step until the next call. Every rank must set the same values: they are not
 * compared across ranks. Returns SIGLIP_ERR_INVALID for values out of range (NaN included) and SIGLIP_ERR_STATE
 * outside the mode.
 */
int siglip_set_focal(siglip_ctx* ctx, float gamma, float alpha);

/*
 * In-batch retrieval metrics of the NEXT siglip_fwd_bwd(_scaled) / siglip_forward / siglip_fwd call (that step only),
 * computed from the logits the loss kernels already hold in registers, without a second similarity GEMM:
 *   i2t_index[i] = argmax_j s_ij over all sum(T) texts, for each of this rank's B images (global text index; with hard
 *                  negatives a winning extra is a miss)
 *   t2i_index[j] = argmax_i s_ij over all sum(R) images, for each of this rank's B paired texts (global image index;
 *                  under SIGLIP_OPT_EXTRA_TEXT_IDS for each of its T texts, so t2i_index is then [T]). A winning extra
 *                  image is a miss unless SIGLIP_OPT_EXTRA_IMAGE_IDS is on and its id is the text's
 *   With extra images, i2t ranks the B paired images ([B]), or under SIGLIP_OPT_EXTRA_IMAGE_IDS all R images ([R]:
 *                  an extra image whose id matches no text is always an i2t miss)
 *   top1[0] / top1[1] = fraction of this rank's images / texts whose top-1 is a positive: the positional diagonal, or
 *                       under SIGLIP_OPT_SAMPLE_IDS a pair with the same id, on any rank. Under
 *                       SIGLIP_OPT_EXTRA_TEXT_IDS an extra with the image's id is a hit for i2t, and top1[1] counts
 *                       over all T texts: an extra whose id matches no image is always a t2i miss
 * Global indices follow the concatenated batch (prefix sums of the per-rank image / text counts). Ties go to the lowest global index;
 * the ranking uses the kernel's fp32 <img, txt> (z = exp(t') s + b is monotone in s). Per rank, like the loss.
 * top1: 2 fp32 device floats (required); i2t_index / t2i_index: [B] int64 device buffers or NULL. Loss and gradients are
 * bit-identical to the same step without metrics. Cost: the step's loss kernels run an instantiation that also reduces
 * the argmax keys, plus two launches (a memset of the keys and a one-block finalisation kernel). This call only records
 * the pointers and reads nothing on the host, so a single-rank metrics step can be captured into a CUDA graph. On a
 * single-rank context the first call allocates the key buffers (4 x B 64-bit words; also allowed inside a capture), so a
 * context that never asks for metrics holds exactly the workspace it held before.
 * Collective: every rank arms the same steps. The host-buffer entries return SIGLIP_ERR_STATE while armed.
 * A step entry (siglip_fwd_bwd(_scaled) / siglip_forward / siglip_fwd) that returns an error disarms every request
 * (metrics, per-sample losses, top-K). A call refused before the step starts (an argument, the sigma budget, a missing
 * input) writes none of the buffers, and no later step does; an error after the step has started (a launch, a
 * workspace allocation, a peer wait) may leave the buffers written in part. siglip_backward takes no request: a
 * refused backward leaves the requests armed for the next forward.
 */
int siglip_request_metrics(siglip_ctx* ctx, float* top1, int64_t* i2t_index, int64_t* t2i_index);

/* Per-sample losses of the NEXT siglip_fwd_bwd(_scaled) / siglip_forward / siglip_fwd only (detached statistics, fp32):
 *   image_loss[i] (i < R: paired images, then extra images) = sum over every text of the global batch (all ranks,
 *                 hard negatives / extra texts included) of w_ij * l_ij
 *   text_loss[j]  (j < T: paired texts, then extras)        = sum over every image of the global batch (all ranks,
 *                 extra images included) of w_ij * l_ij
 * where l_ij = softplus(-y_ij z_ij) is exactly the pair's term of the loss, with the labels the options give, and w_ij
 * its weight (1 without SIGLIP_OPT_SAMPLE_WEIGHTS). No 1/B: the rank's loss is image_loss.sum() / B up to rounding, and
 * a sample of weight 0 reports exactly 0. Each partial (a 128-column tile of a row, a 16-row slab of a column) is added
 * as a 64-bit fixed-point number (value * 2^32), so the results are bitwise reproducible whatever the cluster shape,
 * stage count, schedule or order of the atomics. A partial that is not finite or not below 2^16 makes its sample
 * report +inf (NaN for a NaN term).
 * image_loss: [R] fp32 device buffer, text_loss: [T] fp32 device buffer, both required. Loss, gradients and the
 * retrieval metrics are bit-identical to the same step without the request.
 * Cost: the step's loss kernels run their own instantiation (kModeSampleLoss), which also adds the row and column sums,
 * plus two launches (a memset of the step's fixed-point words and a one-block finalisation kernel). Workspace: two
 * parities of [world * Tmax + Rmax] sums plus as many poison words, 64-bit each; on a single-rank context
 * 32 * (T + R) bytes allocated by the first call (also allowed inside a capture), on a multi-rank context part of the
 * exported text allocation from creation. This call only records the pointers, so a single-rank step stays capturable.
 * Collective: every rank arms the same steps. Under SIGLIP_OPT_DISTILL the sums are those of the distillation
 * terms; a siglip_ctx_create_distill context returns SIGLIP_ERR_STATE there (siglip_ctx_create_distill_extras takes
 * them). The host-buffer entries return SIGLIP_ERR_STATE while armed. A refused step disarms the request, as for
 * siglip_request_metrics. */
int siglip_request_sample_losses(siglip_ctx* ctx, float* image_loss, float* text_loss);

/* Largest K of siglip_request_topk. */
#define SIGLIP_TOPK_MAX 10

/* Top-K in-batch retrieval of the NEXT siglip_fwd_bwd(_scaled) / siglip_forward / siglip_fwd only (detached):
 *   i2t_topk[i, s] (i < the images siglip_request_metrics ranks) = global index of image i's (s+1)-th best text over
 *                  the global batch, t2i_topk[j, s] the same for text j's images; -1 past the candidates there are
 *   recall[k - 1] (k = 1 .. K) = fraction of those images with a hit among their first k texts, recall[K + k - 1] the
 *                  same for the texts (hits as in siglip_request_metrics: the pair, a shared id, extras by their ids)
 * The ranking is the metrics' own: the key (order-preserving bits of s) << 32 | (0xFFFFFFFF - global index), so ties
 * go to the lower index, recall[0] / recall[K] equal the top-1 rates bit for bit, column 0 equals the top-1 indices,
 * and the lists for K are the first K entries of the lists for any larger K. Bitwise reproducible whatever the cluster
 * shape, stage count, schedule, row panels or order of the atomics.
 * k in 1 .. SIGLIP_TOPK_MAX; recall: [2k] fp32 device buffer (required), i2t_topk [ni, k] and t2i_topk [nt, k] int64
 * device buffers or NULL. Loss, gradients, the retrieval metrics and the per-sample losses are bit-identical to the same
 * step without the request; composes with siglip_request_metrics and siglip_request_sample_losses.
 * Cost: k = 1 runs the metrics path. k > 1 runs the step's loss kernels in their own instantiation, which inserts
 * every logit above a list's current K-th key into per-row and per-column sorted lists, plus two memsets and a
 * one-block finalisation kernel. Workspace: two parities of [world * Tmax] column lists and [Rmax] row lists of
 * SIGLIP_TOPK_MAX 64-bit keys each; the row lists (and on a single-rank context the column lists) are allocated by the
 * first call (also allowed inside a capture), the column lists of a multi-rank context are part of the exported text
 * allocation from creation. This call only records the pointers.
 * Collective: every rank arms the same steps with the same k. Returns SIGLIP_ERR_INVALID for k out of range or a null
 * recall, SIGLIP_ERR_STATE under SIGLIP_OPT_DISTILL on a siglip_ctx_create_distill context (a
 * siglip_ctx_create_distill_extras context takes it); the host-buffer entries return SIGLIP_ERR_STATE while armed.
 * A refused step disarms the request, as for siglip_request_metrics. */
int siglip_request_topk(siglip_ctx* ctx, int k, float* recall, int64_t* i2t_topk, int64_t* t2i_topk);

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
 * These entries take no sample ids or weights: under SIGLIP_OPT_SAMPLE_IDS or SIGLIP_OPT_SAMPLE_WEIGHTS they return
 * SIGLIP_ERR_STATE. They stage [B, D] text and images:
 * on a context with hard negatives (siglip_ctx_create_texts, some T_p != B_p) or extra images (siglip_ctx_create_extras,
 * some R_p != B_p) they return SIGLIP_ERR_STATE.
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

/*
 * Test hook: clusters of the persistent grid that a gradient-kernel launch (SIGLIP_OPT_CTA_GROUP cta_group,
 * SIGLIP_OPT_MCAST mcast, column tiles tile_n = 128 or 256, SIGLIP_OPT_STAGES_GRAD stages = 0, 4 or 6; 256-column
 * tiles always run 4 stages) gets on `device`: the runtime's co-resident clusters of that instantiation, at most
 * SMs / cluster size. Split-K (SIGLIP_OPT_SPLIT_K) cuts the ragged last wave of that grid. Returns the count, or minus
 * the status code.
 */
int siglip_debug_max_active_clusters(int device, int cta_group, int mcast, int tile_n, int stages);

/* Test hook: the same for the loss kernel of one mode (0 the plain loss kernel, whatever its ids, metrics and weights;
 * 2 distillation, 3 per-sample losses, 4 top-K, 5 excluded groups, 6 label sets, 7 focal terms, 8 distillation with
 * options) at SIGLIP_OPT_STAGES_LOSS stages = 0, 4 or 6 (the distillation modes always run 4): the clusters of its
 * persistent grid before a launch caps them at its tiles. Returns the count, or minus the status code.
 */
int siglip_debug_loss_max_active_clusters(int device, int cta_group, int mcast, int mode, int stages);

/* Same contraction launched `iters` times back to back (after one warm-up when iters > 1); *ms_per_iter receives
 * the CUDA-event time per launch. Used to tune the mainloop apart from the loss epilogue. */
int siglip_debug_gemm_timed(int device, int cta_group, int M, int N, int K, const void* A, long long lda, int a_mn,
                            const void* Bm, long long ldb, int b_mn, float* C, long long ldc, int iters,
                            float* ms_per_iter, void* cuda_stream);

/*
 * Test hooks for exercising the multi-chunk schedule of ONE rank on ONE GPU (world > 1 context, no peers):
 * loopback wires every "peer" pointer to stand-in buffers of the context. The peers' exported text allocations are
 * one stand-in with the same layout, peer o's chunk at slot o: siglip_debug_set_text_chunk and its twins below write a
 * peer's chunk (text, ids, groups, label sets, weights, teacher text) there, and every step pulls it into the gathered
 * buffers the kernels read, as from a real owner (the own chunk is written in place, and the step overwrites it with
 * its own inputs). The peers' contribution slots are one [T of this rank, D] fp32 block per peer, zero until
 * siglip_debug_set_peer_contribution seeds it: the step folds each peer's block into the dtxt OUTPUT, which is then this
 * rank's own-chunk contribution plus the seeded blocks. The test runs the step and reads this rank's per-owner dtxt
 * contributions back: slot c for c != rank (siglip_debug_get_slot), the dtxt output for the own chunk. Chunks and
 * slots hold T_chunk rows (its batch plus its hard negatives).
 */
int siglip_debug_loopback(siglip_ctx* ctx);
int siglip_debug_set_text_chunk(siglip_ctx* ctx, int chunk, const void* txt_dev, void* cuda_stream);
/* Loopback only: the contribution to this rank's text gradient standing in for peer rank `peer`'s ([T of this rank, D]
 * fp32 device buffer, already scaled by the upstream gradient as a peer's gradient kernel writes it). It stays until
 * seeded again, and the step's dtxt output adds it to g x (own contribution). */
int siglip_debug_set_peer_contribution(siglip_ctx* ctx, int peer, const float* contrib_dev, void* cuda_stream);

/* The teacher twin of siglip_debug_set_text_chunk (SIGLIP_OPT_DISTILL): the teacher text of chunk `chunk`
 * ([T of that rank, D_teacher] in the teacher's format: paired texts, then extras) as its owner would have published
 * it. */
int siglip_debug_set_teacher_text_chunk(siglip_ctx* ctx, int chunk, const void* ttxt_dev, void* cuda_stream);

/* The teacher's operand formats (width D_teacher): siglip_convert_f32_rows and siglip_normalize_fwd_rows over `rows`
 * rows of teacher embeddings, with the format given by f16 (1: fp16(16 x), 0: bf16). Forward only. */
int siglip_teacher_convert_f32(siglip_ctx* ctx, int rows, const float* x_f32, void* out_16bit, int f16,
                               void* cuda_stream);
int siglip_teacher_normalize_fwd(siglip_ctx* ctx, int rows, const void* x, int in_bf16, void* xhat, float* inv_norm,
                                 int f16, void* cuda_stream);
int siglip_debug_get_slot(siglip_ctx* ctx, int chunk, float* out_dev, void* cuda_stream);
/* The ids twin of siglip_debug_set_text_chunk (SIGLIP_OPT_SAMPLE_IDS): the sample ids of text chunk `chunk`
 * ([batch of that rank] int64 device buffer: its paired texts only; [T of that rank] under SIGLIP_OPT_EXTRA_TEXT_IDS:
 * its paired texts, then its extras) as the "peer" would have published them. */
int siglip_debug_set_chunk_ids(siglip_ctx* ctx, int chunk, const int64_t* ids_dev, void* cuda_stream);
/* The groups twin (SIGLIP_OPT_EXCLUDE_GROUPS): the text groups of chunk `chunk` ([T of that rank] int64 device buffer)
 * as the "peer" would have published them. */
int siglip_debug_set_chunk_groups(siglip_ctx* ctx, int chunk, const int64_t* groups_dev, void* cuda_stream);
/* The label-set twin (SIGLIP_OPT_LABEL_SETS): the text sets of chunk `chunk` ([T of that rank, M] int64 device buffer:
 * its paired texts' sets, then its extras') as the "peer" would have published them. */
int siglip_debug_set_chunk_label_sets(siglip_ctx* ctx, int chunk, const int64_t* sets_dev, void* cuda_stream);
/* The weights twin (SIGLIP_OPT_SAMPLE_WEIGHTS): the text weights of chunk `chunk` ([T of that rank] fp32 device buffer,
 * or NULL = ones), clamped like siglip_set_sample_weights, as the "peer" would have published them. */
int siglip_debug_set_chunk_weights(siglip_ctx* ctx, int chunk, const float* text_w_dev, void* cuda_stream);
/* Loopback only: seed the (dt_prime, dbias) mailbox standing in for peer rank `peer`, so that the mean computed under
 * SIGLIP_OPT_SYNC_SCALAR_GRADS can be checked against numbers the kernel did not produce itself. */
int siglip_debug_set_mailbox(siglip_ctx* ctx, int peer, float dt_prime, float dbias);
/* Loopback only: seed the column argmax partials of this rank's text chunk that stand in for peer rank `peer`'s
 * ([B] 64-bit keys, [T] under SIGLIP_OPT_EXTRA_TEXT_IDS or SIGLIP_OPT_LABEL_SETS: (order-preserving fp32 bits of
 * s) << 32 | (0xFFFFFFFF - global image index), 0 = no candidate), so that the cross-rank combine of a metrics step
 * sees candidates the kernel did not produce itself. */
int siglip_debug_set_peer_metric_keys(siglip_ctx* ctx, int peer, const uint64_t* keys_dev, void* cuda_stream);
/* Loopback only: seed the top-K column lists of this rank's text chunk that stand in for peer rank `peer`'s
 * ([T, SIGLIP_TOPK_MAX] 64-bit keys as in siglip_debug_set_peer_metric_keys, each row sorted best first and 0-padded),
 * so that the cross-rank merge of a top-K step sees lists the kernel did not produce itself. */
int siglip_debug_set_peer_topk_keys(siglip_ctx* ctx, int peer, const uint64_t* keys_dev, void* cuda_stream);
/* Loopback only: seed the per-sample-loss column partials of this rank's text chunk that stand in for peer rank
 * `peer`'s ([T] 64-bit fixed-point words, value * 2^32), so that the cross-rank sum of a per-sample-loss step adds
 * numbers the kernel did not produce itself. */
int siglip_debug_set_peer_sample_loss_partials(siglip_ctx* ctx, int peer, const int64_t* partials_dev,
                                               void* cuda_stream);
/* Loopback only: seed the poison words that go with those partials ([T] 64-bit words, bit 0: a partial that was +inf
 * or not below 2^16, bit 1: a NaN partial; 0: none), so that the cross-rank OR of a per-sample-loss step sees poison the
 * kernel did not produce itself. They stay until seeded again. */
int siglip_debug_set_peer_sample_loss_poison(siglip_ctx* ctx, int peer, const int64_t* poison_dev, void* cuda_stream);
/* Loopback only (SIGLIP_OPT_EXTRA_IMAGE_IDS): seed the extra-image ids that stand in for what peer rank `peer` publishes
 * in a metrics step ([R_peer - B_peer] int64 device buffer), so that a t2i winner among its extra images is judged by
 * ids the test chose. */
int siglip_debug_set_peer_extra_image_ids(siglip_ctx* ctx, int peer, const int64_t* ids_dev, void* cuda_stream);
/* The label-set twin: the sets of rank `peer`'s extra images ([E_peer, M] int64 device buffer) as that peer would have
 * published them for a metrics or top-K step (SIGLIP_OPT_LABEL_SETS). */
int siglip_debug_set_peer_extra_image_label_sets(siglip_ctx* ctx, int peer, const int64_t* sets_dev, void* cuda_stream);
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
