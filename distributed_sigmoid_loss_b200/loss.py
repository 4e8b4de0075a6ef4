"""Host-side mirror of the reference's module surface over the sm_90a C-ABI library.

Reference interface (ahmdtaha/distributed_sigmoid_loss):
  * ``DDPSigmoidLoss(gpu_batch_size).forward(image_embeddings, text_embeddings)``
    (distributed_sigmoid_loss.py:8-48) with learnable ``t_prime`` / ``bias`` (:11-12),
  * ``SigLipLoss(cache_labels, rank, world_size, bidir, use_horovod).forward(image_features,
    text_features, logit_scale, logit_bias, output_dict=False)`` (rwightman_sigmoid_loss.py:23-30, 68).

Same names, same argument meaning, same error behaviour (``RuntimeError`` when the batch does not match
``gpu_batch_size``). The arithmetic runs in ``libsiglip_b200.so`` only: PyTorch supplies device memory,
the stream and the process group used to exchange CUDA-IPC handles once. No CPU path exists here.
"""
from __future__ import annotations

import ctypes
import math
from typing import Dict, Optional, Tuple

import torch
import torch.distributed as dist
import torch.nn as nn

from . import _capi

# Largest K of the top-K in-batch retrieval (SIGLIP_TOPK_MAX in include/siglip_b200.h)
TOPK_MAX = 10
# labels per set at most (SIGLIP_MAX_LABELS): multi_label=M takes 1 <= M <= MAX_LABELS
MAX_LABELS = 4


def _group_rank_world(group) -> Tuple[int, int]:
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(group), dist.get_world_size(group)
    return 0, 1


def chunk_schedule(rank: int, world: int, bidir: bool = False):
    """Order in which a rank scores its images against the text chunks (owner rank per step), own chunk first.
    bidir=False: rank+1, rank+2, ... (mod world) — the pairs of the reference's unidirectional ring
    (rwightman_sigmoid_loss.py:108-122 receives from the left neighbour, i.e. rank-1, rank-2, ...; the set of
    (image-rank, text-chunk) pairs covered is identical, only the direction differs).
    bidir=True: rank+1, rank-1, rank+2, rank-2, ... — the order of its bidirectional exchange (:75-107).
    Either way every owner is read by exactly one rank at every step (mirrors step_owner() in csrc/siglip_capi.cu)."""
    def offset(k):
        if not bidir:
            return k
        return (k + 1) // 2 if (k & 1) else -(k // 2)
    return [(rank + offset(k)) % world for k in range(world)]


class SigmoidLossEngine:
    """Owns one ``siglip_ctx`` (workspaces + peer mappings) for a fixed (device, B, D, process group)."""

    def __init__(self, batch: int, dim: int, device: torch.device, group=None, cta_group: int = 2,
                 overlap_pull: bool = True, rank_world: Optional[Tuple[int, int]] = None, loopback: bool = False,
                 batch_per_rank=None, texts_per_rank=None, images_per_rank=None, teacher_dim: int = 0,
                 labels: int = 0, distill_options: bool = False):
        self._L = _capi.lib()
        if not torch.cuda.is_available() or self._L.siglip_device_count() == 0:
            raise RuntimeError("distributed_sigmoid_loss_b200 needs an sm_90 (H100) device; there is no CPU fallback")
        self.batch, self.dim, self.device, self.group = batch, dim, torch.device(device), group
        self.rank, self.world = rank_world if rank_world is not None else _group_rank_world(group)
        h = ctypes.c_void_p()
        self.teacher_dim = int(teacher_dim)
        self.labels = int(labels)   # labels per set of a label-set engine (siglip_ctx_create_labels), 0: none
        # distill_options: a teacher together with extras, label sets, per-sample losses, top-K and groups
        # (siglip_ctx_create_distill_extras); without it a distillation engine refuses them, as it always has
        if distill_options and not self.teacher_dim:
            raise RuntimeError("distill_options=True needs teacher_dim > 0")
        if self.teacher_dim and not distill_options and (images_per_rank is not None or texts_per_rank is not None):
            raise RuntimeError("a distillation engine (teacher_dim > 0) takes no extra texts or images without "
                               "distill_options=True")
        if self.labels and self.teacher_dim and not distill_options:
            raise RuntimeError("a label-set engine (labels > 0) takes no teacher without distill_options=True")
        if distill_options:
            # every text and image of a rank has a teacher row
            bpr, ipr, tpr = self._extras_lists(batch, batch_per_rank, images_per_rank, texts_per_rank)
            _capi.check(self._L.siglip_ctx_create_distill_extras(
                ctypes.byref(h), self.device.index or 0, self.rank, self.world, (ctypes.c_int * self.world)(*bpr),
                (ctypes.c_int * self.world)(*ipr), (ctypes.c_int * self.world)(*tpr), dim, self.teacher_dim,
                self.labels))
            self.batch_per_rank, self.images_per_rank, self.texts_per_rank = bpr, ipr, tpr
            images_per_rank, texts_per_rank = ipr, tpr
        elif self.labels:
            # label sets: the sets' width is part of the exported allocation (siglip_ctx_create_labels)
            bpr, ipr, tpr = self._extras_lists(batch, batch_per_rank, images_per_rank, texts_per_rank)
            _capi.check(self._L.siglip_ctx_create_labels(ctypes.byref(h), self.device.index or 0, self.rank, self.world,
                                                         (ctypes.c_int * self.world)(*bpr),
                                                         (ctypes.c_int * self.world)(*ipr),
                                                         (ctypes.c_int * self.world)(*tpr), dim, self.labels))
            self.batch_per_rank, self.images_per_rank, self.texts_per_rank = bpr, ipr, tpr
            images_per_rank, texts_per_rank = ipr, tpr
        elif self.teacher_dim:
            # distillation: the teacher width is part of the exported allocation (siglip_ctx_create_distill)
            bpr = [int(b) for b in batch_per_rank] if batch_per_rank is not None else [batch] * self.world
            if len(bpr) != self.world or bpr[self.rank] != batch:
                raise RuntimeError(f"batch_per_rank {bpr} must list one batch per rank and hold {batch} at rank {self.rank}")
            _capi.check(self._L.siglip_ctx_create_distill(ctypes.byref(h), self.device.index or 0, self.rank, self.world,
                                                          (ctypes.c_int * self.world)(*bpr), dim, self.teacher_dim))
            self.batch_per_rank = bpr
        elif images_per_rank is not None:
            # extra images: rank p holds images_per_rank[p] >= its batch images, the paired ones first, then its extras
            # (siglip_ctx_create_extras); every rank passes the same three lists
            bpr, ipr, tpr = self._extras_lists(batch, batch_per_rank, images_per_rank, texts_per_rank)
            _capi.check(self._L.siglip_ctx_create_extras(ctypes.byref(h), self.device.index or 0, self.rank, self.world,
                                                         (ctypes.c_int * self.world)(*bpr),
                                                         (ctypes.c_int * self.world)(*ipr),
                                                         (ctypes.c_int * self.world)(*tpr), dim))
            self.batch_per_rank, self.images_per_rank, self.texts_per_rank = bpr, ipr, tpr
        elif texts_per_rank is not None:
            # hard-negative captions: rank p holds texts_per_rank[p] >= its batch texts, the paired ones first, then its
            # extras (siglip_ctx_create_texts); every rank passes the same lists
            bpr = [int(b) for b in batch_per_rank] if batch_per_rank is not None else [batch] * self.world
            tpr = [int(t) for t in texts_per_rank]
            if len(bpr) != self.world or bpr[self.rank] != batch or len(tpr) != self.world:
                raise RuntimeError(f"batch_per_rank {bpr} / texts_per_rank {tpr} must list one entry per rank and hold "
                                   f"batch {batch} at rank {self.rank}")
            if any(t < b for t, b in zip(tpr, bpr)):
                raise RuntimeError(f"texts_per_rank {tpr} must be >= batch_per_rank {bpr} on every rank")
            _capi.check(self._L.siglip_ctx_create_texts(ctypes.byref(h), self.device.index or 0, self.rank, self.world,
                                                        (ctypes.c_int * self.world)(*bpr),
                                                        (ctypes.c_int * self.world)(*tpr), dim))
            self.batch_per_rank, self.texts_per_rank = bpr, tpr
        elif batch_per_rank is not None:
            # extension (SURVEY.md §8f-4): ranks with different batch sizes; every rank passes the same list
            bpr = [int(b) for b in batch_per_rank]
            if len(bpr) != self.world or bpr[self.rank] != batch:
                raise RuntimeError(f"batch_per_rank {bpr} must list one batch per rank and hold {batch} at rank {self.rank}")
            arr = (ctypes.c_int * self.world)(*bpr)
            _capi.check(self._L.siglip_ctx_create_uneven(ctypes.byref(h), self.device.index or 0, self.rank, self.world,
                                                         arr, dim))
            self.batch_per_rank = bpr
        else:
            _capi.check(self._L.siglip_ctx_create(ctypes.byref(h), self.device.index or 0, self.rank, self.world,
                                                  batch, dim))
            self.batch_per_rank = [batch] * self.world
        if texts_per_rank is None:
            self.texts_per_rank = list(self.batch_per_rank)
        if images_per_rank is None:
            self.images_per_rank = list(self.batch_per_rank)
        self.texts = self.texts_per_rank[self.rank]   # rows of txt / dtxt: the batch plus this rank's hard negatives
        self.images = self.images_per_rank[self.rank]   # rows of img / dimg: the batch plus this rank's extra images
        self.extra_text_ids = False   # SIGLIP_OPT_EXTRA_TEXT_IDS: every text of a chunk carries an id (see set_option)
        self.extra_image_ids = False  # SIGLIP_OPT_EXTRA_IMAGE_IDS: every image of this rank carries an id
        self.label_sets = False       # SIGLIP_OPT_LABEL_SETS: every sample, extra text and extra image carries a set
        self._h = h
        _capi.check(self._L.siglip_ctx_set_option(h, _capi.SIGLIP_OPT_CTA_GROUP, int(cta_group)))
        _capi.check(self._L.siglip_ctx_set_option(h, _capi.SIGLIP_OPT_OVERLAP_PULL, int(bool(overlap_pull))))
        if self.world > 1:
            if loopback:  # single-GPU test mode: one rank of a W-rank job, peers wired to local buffers
                _capi.check(self._L.siglip_debug_loopback(h))
            else:
                self._exchange_handles()

    def _extras_lists(self, batch: int, batch_per_rank, images_per_rank, texts_per_rank):
        """(batch_per_rank, images_per_rank, texts_per_rank) of an engine created with extras or label sets: one entry
        per rank (None: the batch on every rank, and no extras), this rank's batch at its index, and images and texts
        at least the batch on every rank."""
        bpr = [int(b) for b in batch_per_rank] if batch_per_rank is not None else [batch] * self.world
        ipr = [int(r) for r in images_per_rank] if images_per_rank is not None else list(bpr)
        tpr = [int(t) for t in texts_per_rank] if texts_per_rank is not None else list(bpr)
        if len(bpr) != self.world or bpr[self.rank] != batch or len(ipr) != self.world or len(tpr) != self.world:
            raise RuntimeError(f"batch_per_rank {bpr} / images_per_rank {ipr} / texts_per_rank {tpr} must list one "
                               f"entry per rank and hold batch {batch} at rank {self.rank}")
        if any(r < b for r, b in zip(ipr, bpr)) or any(t < b for t, b in zip(tpr, bpr)):
            raise RuntimeError(f"images_per_rank {ipr} and texts_per_rank {tpr} must be >= batch_per_rank {bpr} on "
                               f"every rank")
        return bpr, ipr, tpr

    # -- peer bootstrap: replaces the reference's reliance on the process group for every step ------------
    def _exchange_handles(self) -> None:
        n = int(self._L.siglip_ctx_handle_bytes())
        buf = ctypes.create_string_buffer(n)
        _capi.check(self._L.siglip_ctx_export_handles(self._h, buf, n))
        blobs = [None] * self.world
        dist.all_gather_object(blobs, bytes(buf.raw), group=self.group)
        joined = b"".join(blobs)
        _capi.check(self._L.siglip_ctx_import_handles(self._h, joined, n))
        dist.barrier(group=self.group)

    def set_option(self, option: int, value: int) -> None:
        _capi.check(self._L.siglip_ctx_set_option(self._h, option, value))
        if option == _capi.SIGLIP_OPT_EXTRA_TEXT_IDS or (option == _capi.SIGLIP_OPT_SAMPLE_IDS and not value):
            self.extra_text_ids = bool(value)   # the library clears the extras' ids with the sample ids
        if option == _capi.SIGLIP_OPT_EXTRA_IMAGE_IDS or (option == _capi.SIGLIP_OPT_SAMPLE_IDS and not value):
            self.extra_image_ids = bool(value)
        if option == _capi.SIGLIP_OPT_LABEL_SETS:
            self.label_sets = bool(value)

    def set_sigma_budget(self, sigma_budget_bytes: Optional[int]) -> None:
        """SIGLIP_OPT_SIGMA_BUDGET_MIB: bound the 16-bit sigma operands to sigma_budget_bytes (rounded down to MiB; None
        or 0: unbounded). Fused steps then run in row panels (see the option in include/siglip_b200.h)."""
        mib = _sigma_budget_mib(sigma_budget_bytes)
        self.set_option(_capi.SIGLIP_OPT_SIGMA_BUDGET_MIB, mib)
        self.sigma_budget_mib = mib

    def split_fits_budget(self) -> bool:
        """Whether the split forward / backward (W whole sigma operands kept until the backward) fits the budget."""
        return self.sigma_panels(self.world)[2]

    def sigma_panels(self, buffers: int = 0) -> Tuple[int, int, bool]:
        """(panel rows, panels, whole) of the budget for `buffers` sigma operands (0: the fused step's); panel rows 0
        means the budget is below one minimal panel, whole that it holds the whole operands (siglip_ctx_sigma_panels)."""
        rows, n, whole = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        _capi.check(self._L.siglip_ctx_sigma_panels(self._h, int(buffers), ctypes.byref(rows), ctypes.byref(n),
                                                    ctypes.byref(whole)))
        return rows.value, n.value, bool(whole.value)

    def kernel_times(self):
        """(loss_ms, loss_launches, grad_ms, grad_launches) since the last call; needs SIGLIP_OPT_KERNEL_TIMING."""
        lm, gm = ctypes.c_double(), ctypes.c_double()
        ln, gn = ctypes.c_int(), ctypes.c_int()
        _capi.check(self._L.siglip_ctx_kernel_times(self._h, ctypes.byref(lm), ctypes.byref(ln), ctypes.byref(gm),
                                                    ctypes.byref(gn)))
        return lm.value, ln.value, gm.value, gn.value

    def debug_set_text_chunk(self, chunk: int, txt: torch.Tensor) -> None:
        _capi.check(self._L.siglip_debug_set_text_chunk(self._h, chunk, txt.data_ptr(), self._stream()))

    def set_teacher(self, timg: torch.Tensor, ttxt: torch.Tensor, t_prime: torch.Tensor, bias: torch.Tensor,
                    lam: float) -> None:
        """SIGLIP_OPT_DISTILL: the teacher of the NEXT step. timg: [images, teacher_dim], ttxt: [texts, teacher_dim]
        (paired rows, then extras, like the student's), contiguous, 16-byte aligned, both bf16 or both float16 holding
        16*x (see teacher_operand); t_prime / bias: 1-element fp32 tensors on the engine's device (t_T = exp(t_prime));
        lam in (0, 1]. Only the pointers are recorded: the tensors must stay alive until the step is enqueued."""
        for x, rows in ((timg, self.images), (ttxt, self.texts)):
            if x.device != self.device or x.dtype not in (torch.bfloat16, torch.float16) or not x.is_contiguous() or \
                    tuple(x.shape) != (rows, self.teacher_dim):
                raise RuntimeError(f"teacher operands must be contiguous bf16 (or fp16 x16) [{rows}, "
                                   f"{self.teacher_dim}] tensors on {self.device}, got {tuple(x.shape)} {x.dtype}")
        if timg.dtype != ttxt.dtype:
            raise RuntimeError("teacher image and text operands must use the same 16-bit format")
        for x in (t_prime, bias):
            if x.dtype != torch.float32 or x.numel() != 1 or x.device != self.device:
                raise RuntimeError("teacher scalars must be 1-element fp32 tensors on the engine's device")
        _capi.check(self._L.siglip_set_teacher(self._h, timg.data_ptr(), ttxt.data_ptr(),
                                               int(timg.dtype == torch.float16), t_prime.data_ptr(), bias.data_ptr(),
                                               float(lam)))

    def teacher_operand(self, x: torch.Tensor, normalize: bool) -> torch.Tensor:
        """A teacher embedding [B, teacher_dim] in the kernels' operand format, by the student's rules: bf16 as it is,
        anything else through the fp32 conversion to float16 holding 16*x; normalize=True L2-normalises it first."""
        hi = x.dtype != torch.bfloat16
        if normalize:
            if x.dtype not in (torch.float32, torch.bfloat16):
                x = x.float()
            x = _aligned(x)
            out = torch.empty(x.shape[0], self.teacher_dim, device=self.device,
                              dtype=torch.float16 if hi else torch.bfloat16)
            inv = torch.empty(x.shape[0], device=self.device, dtype=torch.float32)
            with torch.cuda.device(self.device):
                _capi.check(self._L.siglip_teacher_normalize_fwd(self._h, x.shape[0], x.data_ptr(),
                                                                 int(x.dtype == torch.bfloat16), out.data_ptr(),
                                                                 inv.data_ptr(), int(hi), self._stream()))
            return out
        if not hi:
            return _aligned(x)
        x = _aligned(x.float())
        out = torch.empty(x.shape[0], self.teacher_dim, device=self.device, dtype=torch.float16)
        with torch.cuda.device(self.device):
            _capi.check(self._L.siglip_teacher_convert_f32(self._h, x.shape[0], x.data_ptr(), out.data_ptr(), 1,
                                                           self._stream()))
        return out

    def debug_set_teacher_text_chunk(self, chunk: int, ttxt: torch.Tensor) -> None:
        """Loopback: the teacher text of chunk `chunk` ([T_c, teacher_dim], the teacher's operand format: paired texts,
        then extras) as its owner would have published it."""
        _capi.check(self._L.siglip_debug_set_teacher_text_chunk(self._h, chunk, ttxt.data_ptr(), self._stream()))

    def set_sample_ids(self, ids: torch.Tensor) -> None:
        """SIGLIP_OPT_SAMPLE_IDS: this rank's sample ids ([B] int64, contiguous, on the engine's device) for the NEXT
        step. They are copied on the current stream, so `ids` may be released or overwritten afterwards."""
        self._check_ids(ids, self.batch)
        with torch.cuda.device(self.device):
            _capi.check(self._L.siglip_set_sample_ids(self._h, ids.data_ptr(), self._stream()))

    def set_extra_text_ids(self, ids: torch.Tensor) -> None:
        """SIGLIP_OPT_EXTRA_TEXT_IDS: the ids of this rank's T - B extra texts ([T - B] int64, contiguous, on the engine's
        device) for the NEXT step, copied on the current stream like set_sample_ids."""
        self._check_ids(ids, self.texts - self.batch)
        with torch.cuda.device(self.device):
            _capi.check(self._L.siglip_set_extra_text_ids(self._h, ids.data_ptr(), self._stream()))

    def set_extra_image_ids(self, ids: torch.Tensor) -> None:
        """SIGLIP_OPT_EXTRA_IMAGE_IDS: the ids of this rank's R - B extra images ([R - B] int64, contiguous, on the engine's
        device) for the NEXT step, copied on the current stream like set_sample_ids."""
        self._check_ids(ids, self.images - self.batch)
        with torch.cuda.device(self.device):
            _capi.check(self._L.siglip_set_extra_image_ids(self._h, ids.data_ptr(), self._stream()))

    def debug_set_peer_extra_image_ids(self, peer: int, ids: torch.Tensor) -> None:
        """Loopback: the extra-image ids ([R_peer - B_peer] int64) standing in for what peer `peer` publishes in a
        metrics step."""
        self._check_ids(ids, self.images_per_rank[peer] - self.batch_per_rank[peer])
        _capi.check(self._L.siglip_debug_set_peer_extra_image_ids(self._h, peer, ids.data_ptr(), self._stream()))

    def set_sample_weights(self, image_weights: Optional[torch.Tensor], text_weights: Optional[torch.Tensor]) -> None:
        """SIGLIP_OPT_SAMPLE_WEIGHTS: this rank's image weights ([R] fp32: the paired images, then the extra images) and
        text weights ([T] fp32: the paired texts, then the extras), contiguous on the engine's device, or None for ones,
        for the NEXT step. Copied on the current stream with every value clamped into [0, 1] (NaN -> 0), so the tensors may
        be released or overwritten afterwards."""
        self._check_weights(image_weights, self.images)
        self._check_weights(text_weights, self.texts)
        with torch.cuda.device(self.device):
            _capi.check(self._L.siglip_set_sample_weights(
                self._h, image_weights.data_ptr() if image_weights is not None else None,
                text_weights.data_ptr() if text_weights is not None else None, self._stream()))

    def debug_set_chunk_weights(self, chunk: int, text_weights: Optional[torch.Tensor]) -> None:
        """Loopback: the text weights of chunk `chunk` ([T_c] fp32, or None for ones) as its owner would have published
        them (clamped the same way)."""
        self._check_weights(text_weights, self.texts_per_rank[chunk])
        _capi.check(self._L.siglip_debug_set_chunk_weights(
            self._h, chunk, text_weights.data_ptr() if text_weights is not None else None, self._stream()))

    def _check_weights(self, w: Optional[torch.Tensor], n: int) -> None:
        if w is not None and (w.dtype != torch.float32 or tuple(w.shape) != (n,) or not w.is_contiguous() or
                              w.device != self.device):
            raise RuntimeError(f"sample weights must be a contiguous fp32 [{n}] tensor on {self.device} (or None), got "
                               f"{tuple(w.shape)} {w.dtype} on {w.device}")

    def set_groups(self, image_groups: torch.Tensor, text_groups: torch.Tensor) -> None:
        """SIGLIP_OPT_EXCLUDE_GROUPS: this rank's image groups ([R] int64: the paired images, then the extra images) and
        text groups ([T] int64: the paired texts, then the extras), contiguous on the engine's device, for the NEXT step.
        Copied on the current stream like set_sample_ids; a negative group matches nothing."""
        self._check_ids(image_groups, self.images)
        self._check_ids(text_groups, self.texts)
        with torch.cuda.device(self.device):
            _capi.check(self._L.siglip_set_groups(self._h, image_groups.data_ptr(), text_groups.data_ptr(),
                                                  self._stream()))

    def debug_set_chunk_groups(self, chunk: int, groups: torch.Tensor) -> None:
        """Loopback: the text groups of chunk `chunk` ([T_c] int64) as its owner would have published them."""
        self._check_ids(groups, self.texts_per_rank[chunk])
        _capi.check(self._L.siglip_debug_set_chunk_groups(self._h, chunk, groups.data_ptr(), self._stream()))

    def set_label_sets(self, sample_labels: torch.Tensor, extra_text_labels: Optional[torch.Tensor] = None,
                       extra_image_labels: Optional[torch.Tensor] = None) -> None:
        """SIGLIP_OPT_LABEL_SETS: this rank's label sets for the NEXT step, contiguous int64 on the engine's device:
        sample_labels [B, M] (image i and paired text i), extra_text_labels [T - B, M] and extra_image_labels [R - B, M],
        or None for empty sets. Copied on the current stream like set_sample_ids; a negative entry is an empty slot."""
        self._check_sets(sample_labels, self.batch)
        for x, n in ((extra_text_labels, self.texts - self.batch), (extra_image_labels, self.images - self.batch)):
            if x is not None:
                self._check_sets(x, n)
        with torch.cuda.device(self.device):
            _capi.check(self._L.siglip_set_label_sets(
                self._h, sample_labels.data_ptr(),
                extra_text_labels.data_ptr() if extra_text_labels is not None else None,
                extra_image_labels.data_ptr() if extra_image_labels is not None else None, self._stream()))

    def set_focal(self, gamma: float, alpha: Optional[float] = None) -> None:
        """SIGLIP_OPT_FOCAL: gamma in [0, 8] and alpha in [0, 1] (None: no alpha) of the focal pair loss, for every later
        step until the next call. Host-side only: nothing is launched."""
        _capi.check(self._L.siglip_set_focal(self._h, float(gamma), -1.0 if alpha is None else float(alpha)))

    def debug_set_chunk_label_sets(self, chunk: int, sets: torch.Tensor) -> None:
        """Loopback: the text sets of chunk `chunk` ([T_c, M] int64) as its owner would have published them."""
        self._check_sets(sets, self.texts_per_rank[chunk])
        _capi.check(self._L.siglip_debug_set_chunk_label_sets(self._h, chunk, sets.data_ptr(), self._stream()))

    def debug_set_peer_extra_image_label_sets(self, peer: int, sets: torch.Tensor) -> None:
        """Loopback: the extra-image sets ([R_peer - B_peer, M] int64) standing in for what peer `peer` publishes in a
        metrics or top-K step."""
        self._check_sets(sets, self.images_per_rank[peer] - self.batch_per_rank[peer])
        _capi.check(self._L.siglip_debug_set_peer_extra_image_label_sets(self._h, peer, sets.data_ptr(),
                                                                         self._stream()))

    def _check_sets(self, sets: torch.Tensor, n: int) -> None:
        if sets.dtype != torch.int64 or tuple(sets.shape) != (n, self.labels) or not sets.is_contiguous() or \
                sets.device != self.device:
            raise RuntimeError(f"label sets must be a contiguous int64 [{n}, {self.labels}] tensor on {self.device}, "
                               f"got {tuple(sets.shape)} {sets.dtype} on {sets.device}")

    def debug_set_chunk_ids(self, chunk: int, ids: torch.Tensor) -> None:
        """Loopback: the ids of text chunk `chunk` as its owner would have published them: its sample ids ([B_c]), or
        under SIGLIP_OPT_EXTRA_TEXT_IDS the ids of all its texts ([T_c])."""
        self._check_ids(ids, (self.texts_per_rank if self.extra_text_ids else self.batch_per_rank)[chunk])
        _capi.check(self._L.siglip_debug_set_chunk_ids(self._h, chunk, ids.data_ptr(), self._stream()))

    def _check_ids(self, ids: torch.Tensor, n: int) -> None:
        if ids.dtype != torch.int64 or tuple(ids.shape) != (n,) or not ids.is_contiguous() or ids.device != self.device:
            raise RuntimeError(f"sample ids must be a contiguous int64 [{n}] tensor on {self.device}, got "
                               f"{tuple(ids.shape)} {ids.dtype} on {ids.device}")

    def request_metrics(self, top1: torch.Tensor, i2t_index: Optional[torch.Tensor] = None,
                        t2i_index: Optional[torch.Tensor] = None) -> None:
        """Arm the in-batch retrieval metrics of the NEXT step (siglip_request_metrics): top1 fp32 [2] (i2t, t2i),
        i2t_index int64 [B] ([R] under SIGLIP_OPT_EXTRA_IMAGE_IDS) and t2i_index int64 [B] ([T] under
        SIGLIP_OPT_EXTRA_TEXT_IDS) (global indices) or None, all contiguous on the engine's device. Nothing is read on the
        host; the step writes them on its stream."""
        bufs = ((top1, torch.float32, 2), (i2t_index, torch.int64, self.metric_images),
                (t2i_index, torch.int64, self.metric_texts))
        for k, (x, dt, n) in enumerate(bufs):
            if x is None and k > 0:
                continue
            if x is None or x.dtype != dt or tuple(x.shape) != (n,) or not x.is_contiguous() or x.device != self.device:
                raise RuntimeError(f"metric output {k} must be a contiguous {dt} [{n}] tensor on {self.device}")
        _capi.check(self._L.siglip_request_metrics(self._h, top1.data_ptr(),
                                                   i2t_index.data_ptr() if i2t_index is not None else None,
                                                   t2i_index.data_ptr() if t2i_index is not None else None))

    def debug_set_peer_metric_keys(self, peer: int, keys: torch.Tensor) -> None:
        """Loopback: the column argmax keys ([B] int64 holding the 64-bit key bits, [T] under SIGLIP_OPT_EXTRA_TEXT_IDS)
        standing in for peer `peer`'s partial of this rank's text chunk."""
        n = self.metric_texts
        if keys.dtype != torch.int64 or tuple(keys.shape) != (n,) or not keys.is_contiguous() or \
                keys.device != self.device:
            raise RuntimeError(f"peer metric keys must be a contiguous int64 [{n}] tensor on {self.device}")
        _capi.check(self._L.siglip_debug_set_peer_metric_keys(self._h, peer, keys.data_ptr(), self._stream()))

    def request_topk(self, k: int, recall: torch.Tensor, i2t_topk: Optional[torch.Tensor] = None,
                     t2i_topk: Optional[torch.Tensor] = None) -> None:
        """Arm the top-K in-batch retrieval of the NEXT step (siglip_request_topk), k in 1 .. TOPK_MAX: recall fp32 [2k]
        (i2t recall@1..k, then t2i), i2t_topk int64 [metric_images, k] and t2i_topk int64 [metric_texts, k] (global
        indices, best first, -1 past the candidates) or None, all contiguous on the engine's device. Nothing is read on
        the host; the step writes them on its stream. Refused under distillation without distill_options."""
        if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= TOPK_MAX:
            raise RuntimeError(f"k must be an int in 1 .. {TOPK_MAX}, got {k!r}")
        bufs = (("recall", recall, torch.float32, (2 * k,)),
                ("i2t_topk", i2t_topk, torch.int64, (self.metric_images, k)),
                ("t2i_topk", t2i_topk, torch.int64, (self.metric_texts, k)))
        for name, x, dt, shape in bufs:
            if x is None and name != "recall":
                continue
            if not isinstance(x, torch.Tensor) or x.dtype != dt or tuple(x.shape) != shape or not x.is_contiguous() \
                    or x.device != self.device:
                raise RuntimeError(f"{name} must be a contiguous {dt} {list(shape)} tensor on {self.device}")
        _capi.check(self._L.siglip_request_topk(self._h, k, recall.data_ptr(),
                                                i2t_topk.data_ptr() if i2t_topk is not None else None,
                                                t2i_topk.data_ptr() if t2i_topk is not None else None))

    def debug_set_peer_topk_keys(self, peer: int, keys: torch.Tensor) -> None:
        """Loopback: the top-K column lists ([T, TOPK_MAX] int64 holding the 64-bit keys, each row sorted best first and
        0-padded) standing in for peer `peer`'s lists of this rank's text chunk."""
        shape = (self.texts, TOPK_MAX)
        if keys.dtype != torch.int64 or tuple(keys.shape) != shape or not keys.is_contiguous() or \
                keys.device != self.device:
            raise RuntimeError(f"peer top-K keys must be a contiguous int64 {list(shape)} tensor on {self.device}")
        _capi.check(self._L.siglip_debug_set_peer_topk_keys(self._h, peer, keys.data_ptr(), self._stream()))

    def request_sample_losses(self, image_loss: torch.Tensor, text_loss: torch.Tensor) -> None:
        """Arm the per-sample losses of the NEXT step (siglip_request_sample_losses): image_loss fp32 [R] (the paired
        images, then the extra images) and text_loss fp32 [T] (the paired texts, then the extras), contiguous on the
        engine's device. image_loss[i] is the sum of w_ij softplus(-y_ij z_ij) over every text of the global batch,
        text_loss[j] the same sum over every image of the global batch (no 1/B). Nothing is read on the host; the step
        writes them on its stream. Refused under distillation without distill_options; with it the terms are
        w_ij (softplus(z_ij) - q_ij z_ij)."""
        for name, x, n in (("image_loss", image_loss, self.images), ("text_loss", text_loss, self.texts)):
            if not isinstance(x, torch.Tensor) or x.dtype != torch.float32 or tuple(x.shape) != (n,) or \
                    not x.is_contiguous() or x.device != self.device:
                raise RuntimeError(f"{name} must be a contiguous fp32 [{n}] tensor on {self.device}")
        _capi.check(self._L.siglip_request_sample_losses(self._h, image_loss.data_ptr(), text_loss.data_ptr()))

    def debug_set_peer_sample_loss_partials(self, peer: int, partials: torch.Tensor) -> None:
        """Loopback: the per-sample-loss column partials ([T] int64 fixed-point words, value * 2^32) standing in for peer
        `peer`'s partial of this rank's text chunk."""
        n = self.texts
        if partials.dtype != torch.int64 or tuple(partials.shape) != (n,) or not partials.is_contiguous() or \
                partials.device != self.device:
            raise RuntimeError(f"peer sample-loss partials must be a contiguous int64 [{n}] tensor on {self.device}")
        _capi.check(self._L.siglip_debug_set_peer_sample_loss_partials(self._h, peer, partials.data_ptr(),
                                                                       self._stream()))

    def debug_set_peer_sample_loss_poison(self, peer: int, poison: torch.Tensor) -> None:
        """Loopback: the poison words ([T] int64; 1: a +inf or too large partial, 2: a NaN partial, 0: none) that go with
        peer `peer`'s seeded partials; they stay until seeded again."""
        n = self.texts
        if poison.dtype != torch.int64 or tuple(poison.shape) != (n,) or not poison.is_contiguous() or \
                poison.device != self.device:
            raise RuntimeError(f"peer sample-loss poison must be a contiguous int64 [{n}] tensor on {self.device}")
        _capi.check(self._L.siglip_debug_set_peer_sample_loss_poison(self._h, peer, poison.data_ptr(), self._stream()))

    @property
    def metric_images(self) -> int:
        """Images of this rank that i2t ranks: the paired ones, or all R under SIGLIP_OPT_EXTRA_IMAGE_IDS or
        SIGLIP_OPT_LABEL_SETS."""
        return self.images if (self.extra_image_ids or self.label_sets) else self.batch

    @property
    def metric_texts(self) -> int:
        """Texts of this rank that t2i ranks: the paired ones, or all T under SIGLIP_OPT_EXTRA_TEXT_IDS or
        SIGLIP_OPT_LABEL_SETS."""
        return self.texts if (self.extra_text_ids or self.label_sets) else self.batch

    def debug_get_slot(self, chunk: int) -> torch.Tensor:
        out = torch.empty(self.texts_per_rank[chunk], self.dim, device=self.device, dtype=torch.float32)
        _capi.check(self._L.siglip_debug_get_slot(self._h, chunk, out.data_ptr(), self._stream()))
        return out

    def debug_set_mailbox(self, peer: int, dt_prime: float, dbias: float) -> None:
        _capi.check(self._L.siglip_debug_set_mailbox(self._h, peer, float(dt_prime), float(dbias)))

    def aux_trace(self, max_launches: int = 4096):
        """Per launch since the last call, globaltimer ns: (aux start, flags seen, aux jobs done, launch end, kernel
        entry, set-up done, first operands landed, last MMA issued, first CTA finished, latest / earliest "last MMA issued"
        over the CTAs, last CTA through its tiles, last / first CTA to enter the kernel, last CTA through its set-up, unused);
        needs SIGLIP_OPT_AUX_TRACE."""
        buf = (ctypes.c_ulonglong * (16 * max_launches))()
        n = ctypes.c_int(0)
        _capi.check(self._L.siglip_ctx_aux_trace(self._h, ctypes.cast(buf, ctypes.c_void_p), max_launches,
                                                 ctypes.byref(n)))
        return [tuple(int(buf[16 * i + j]) for j in range(16)) for i in range(n.value)]

    @property
    def workspace_bytes(self) -> int:
        return int(self._L.siglip_ctx_workspace_bytes(self._h))

    @property
    def launch_count(self) -> int:
        return int(self._L.siglip_ctx_launch_count(self._h))

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def fwd_bwd(self, img: torch.Tensor, txt: torch.Tensor, t_prime: torch.Tensor, bias: torch.Tensor,
                grad_dtype: torch.dtype = torch.float32, grad_out: Optional[torch.Tensor] = None):
        """The fused step (siglip_fwd_bwd): loss and gradient kernels alternate chunk by chunk, two sigma operands
        whatever the world size. img/txt: [B, D] bf16 contiguous on self.device; t_prime/bias: fp32 [1]. Returns
        (loss[1], dimg[B,D], dtxt[T,D], dt_prime[1], dbias[1]) for an upstream gradient of 1 (or `grad_out`, a
        1-element fp32 device tensor, multiplied in by the kernel epilogues); scalars are fp32, dimg/dtxt are
        `grad_dtype` (fp32, or bf16 written directly by the kernel epilogue). txt is [T, D]: T = B plus this rank's hard
        negatives (texts_per_rank)."""
        self._check(img, txt)
        self._set_grad_dtype(grad_dtype)
        opts = dict(device=self.device, dtype=torch.float32)
        scal = torch.empty(3, **opts)                 # loss, dt', dbias in one allocation
        loss, dtp, db = scal[0:1], scal[1:2], scal[2:3]
        if self._set_tprime_f64(t_prime):
            dtp = torch.empty(1, device=self.device, dtype=torch.float64)
        dimg = torch.empty(self.images, self.dim, device=self.device, dtype=grad_dtype)
        dtxt = torch.empty(self.texts, self.dim, device=self.device, dtype=grad_dtype)
        with torch.cuda.device(self.device):
            _capi.check(self._L.siglip_fwd_bwd_scaled(
                self._h, img.data_ptr(), txt.data_ptr(), t_prime.data_ptr(), bias.data_ptr(),
                grad_out.data_ptr() if grad_out is not None else None, loss.data_ptr(), dimg.data_ptr(),
                dtxt.data_ptr(), dtp.data_ptr(), db.data_ptr(), self._stream()))
        return loss, dimg, dtxt, dtp, db

    # -- the two halves autograd uses ----------------------------------------------------------------------
    @property
    def saved_generation(self) -> int:
        return int(self._L.siglip_ctx_saved_generation(self._h))

    def forward(self, img: torch.Tensor, txt: torch.Tensor, t_prime: torch.Tensor, bias: torch.Tensor,
                save_for_backward: bool) -> torch.Tensor:
        """The W loss kernels. Returns loss[1] (fp32). With save_for_backward the context keeps the sigma operands."""
        self._check(img, txt)
        self._set_tprime_f64(t_prime)
        loss = torch.empty(1, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            _capi.check(self._L.siglip_forward(self._h, img.data_ptr(), txt.data_ptr(), t_prime.data_ptr(),
                                               bias.data_ptr(), loss.data_ptr(), int(bool(save_for_backward)),
                                               self._stream()))
        return loss

    def backward(self, img: torch.Tensor, txt: torch.Tensor, t_prime: torch.Tensor, grad_out: Optional[torch.Tensor],
                 grad_dtype: torch.dtype = torch.float32):
        """The W gradient kernels on the state saved by the last forward(save_for_backward=True); every gradient is
        multiplied by grad_out (1-element fp32 device tensor, or None for 1) inside the kernel epilogues.
        Returns (dimg, dtxt) in grad_dtype and (dt_prime, dbias) as fp32 [1]."""
        self._check(img, txt)
        self._set_grad_dtype(grad_dtype)
        scal = torch.empty(2, device=self.device, dtype=torch.float32)
        dtp, db = scal[0:1], scal[1:2]
        if self._set_tprime_f64(t_prime):
            dtp = torch.empty(1, device=self.device, dtype=torch.float64)
        dimg = torch.empty(self.images, self.dim, device=self.device, dtype=grad_dtype)
        dtxt = torch.empty(self.texts, self.dim, device=self.device, dtype=grad_dtype)
        with torch.cuda.device(self.device):
            _capi.check(self._L.siglip_backward(self._h, img.data_ptr(), txt.data_ptr(), t_prime.data_ptr(),
                                                grad_out.data_ptr() if grad_out is not None else None,
                                                dimg.data_ptr(), dtxt.data_ptr(), dtp.data_ptr(), db.data_ptr(),
                                                self._stream()))
        return dimg, dtxt, dtp, db

    def _set_grad_dtype(self, grad_dtype: torch.dtype) -> None:
        if grad_dtype not in (torch.float32, torch.bfloat16):
            raise RuntimeError("grad_dtype must be float32 or bfloat16")
        want_bf16 = grad_dtype == torch.bfloat16
        if want_bf16 != getattr(self, "_grad_bf16", False):
            _capi.check(self._L.siglip_ctx_set_option(self._h, _capi.SIGLIP_OPT_GRAD_BF16, int(want_bf16)))
            self._grad_bf16 = want_bf16

    def _rows_ok(self, x: torch.Tensor) -> bool:
        """[B, D] (images, paired texts), [T, D] (texts with this rank's hard negatives) or [R, D] (images with its extra
        images)."""
        return x.dim() == 2 and x.shape[0] in (self.batch, self.texts, self.images) and x.shape[1] == self.dim

    def normalize_fwd(self, x: torch.Tensor, f16: bool = False):
        """F.normalize(x, dim=1) fused with the rounding to the kernels' operand format: returns (xhat [N, D] bf16, or
        float16 holding 16*xhat with f16=True; inv_norm fp32 [N]). x: fp32 or bf16 [N, D] contiguous, N = B or T."""
        if not self._rows_ok(x) or x.dtype not in (torch.float32, torch.bfloat16) or \
                not x.is_contiguous() or x.device != self.device:
            raise RuntimeError(f"normalize_fwd expects a contiguous fp32/bf16 [{self.batch}, {self.texts} or "
                               f"{self.images}, {self.dim}] "
                               f"tensor on {self.device}")
        self._set_input_f16(f16)
        n = x.shape[0]
        xhat = torch.empty(n, self.dim, device=self.device, dtype=torch.float16 if f16 else torch.bfloat16)
        inv = torch.empty(n, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            _capi.check(self._L.siglip_normalize_fwd_rows(self._h, n, x.data_ptr(), int(x.dtype == torch.bfloat16),
                                                          xhat.data_ptr(), inv.data_ptr(), self._stream()))
        return xhat, inv

    def normalize_bwd(self, x: torch.Tensor, inv: torch.Tensor, dxhat: torch.Tensor) -> torch.Tensor:
        """Backward of normalize_fwd: dx = inv * (dxhat - xhat <xhat, dxhat>), in x's dtype."""
        if not self._rows_ok(x) or tuple(dxhat.shape) != tuple(x.shape) or tuple(inv.shape) != (x.shape[0],):
            raise RuntimeError("normalize_bwd expects x / dxhat [N, D] and inv [N] with N = B, T or R")
        dx = torch.empty_like(x)
        with torch.cuda.device(self.device):
            _capi.check(self._L.siglip_normalize_bwd_rows(self._h, x.shape[0], x.data_ptr(),
                                                          int(x.dtype == torch.bfloat16), inv.data_ptr(),
                                                          dxhat.data_ptr(), int(dxhat.dtype == torch.bfloat16),
                                                          dx.data_ptr(), self._stream()))
        return dx

    def scale(self, src: torch.Tensor, g: torch.Tensor) -> torch.Tensor:
        """src * g with g a 1-element fp32 device tensor (grad_output): one fused pass of the C library."""
        if src.dtype not in (torch.float32, torch.bfloat16) or src.device != self.device:
            raise RuntimeError("scale expects an fp32 or bf16 tensor on the engine's device")
        if not src.is_contiguous():
            src = src.contiguous()
        nbytes = src.numel() * src.element_size()
        dst = torch.empty_like(src)
        with torch.cuda.device(self.device):
            _capi.check(self._L.siglip_scale(self._h, src.data_ptr(), dst.data_ptr(), nbytes,
                                             int(src.dtype == torch.bfloat16), g.data_ptr(), self._stream()))
        return dst

    def fwd(self, img: torch.Tensor, txt: torch.Tensor, t_prime: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
        self._check(img, txt)
        self._set_tprime_f64(t_prime)
        loss = torch.empty(1, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            _capi.check(self._L.siglip_fwd(self._h, img.data_ptr(), txt.data_ptr(), t_prime.data_ptr(),
                                           bias.data_ptr(), loss.data_ptr(), self._stream()))
        return loss

    def fwd_bwd_host(self, img_host: torch.Tensor, txt_host: torch.Tensor, t_prime: float, bias: float,
                     dimg_host: Optional[torch.Tensor] = None, dtxt_host: Optional[torch.Tensor] = None):
        """End-to-end step on HOST bf16 buffers (pinned recommended): H2D, step, D2H inside one C call.
        Returns (loss, dt_prime, dbias) as Python floats."""
        self._check_host(img_host, txt_host)
        out = (ctypes.c_float * 3)()
        loss_p = ctypes.cast(out, ctypes.c_void_p).value
        with torch.cuda.device(self.device):
            _capi.check(self._L.siglip_fwd_bwd_host(
                self._h, img_host.data_ptr(), txt_host.data_ptr(), float(t_prime), float(bias), loss_p,
                dimg_host.data_ptr() if dimg_host is not None else None,
                dtxt_host.data_ptr() if dtxt_host is not None else None,
                loss_p + 4, loss_p + 8, self._stream()))
        return float(out[0]), float(out[1]), float(out[2])

    def host_submit(self, img_host: torch.Tensor, txt_host: torch.Tensor, t_prime: float, bias: float,
                    dimg_host: Optional[torch.Tensor] = None, dtxt_host: Optional[torch.Tensor] = None) -> int:
        """Pipelined end-to-end step on HOST bf16 buffers: enqueue this step's host->device copies (internal copy
        stream, two staging sets), the step and the device->host copy of its scalars — and, when `dimg_host` /
        `dtxt_host` (CPU bf16 [B, D], pinned recommended) are given, of its bf16 gradients on a second copy stream;
        returns a ticket for ``host_wait``. At most two steps in flight; the host tensors must stay alive until the
        ticket is waited."""
        self._check_host(img_host, txt_host)
        if (dimg_host is None) != (dtxt_host is None):
            raise RuntimeError("give both gradient host buffers or neither")
        if dimg_host is not None:
            self._check_host(dimg_host, dtxt_host)
        ticket = ctypes.c_ulonglong(0)
        with torch.cuda.device(self.device):
            _capi.check(self._L.siglip_host_submit_grads(
                self._h, img_host.data_ptr(), txt_host.data_ptr(), float(t_prime), float(bias),
                dimg_host.data_ptr() if dimg_host is not None else None,
                dtxt_host.data_ptr() if dtxt_host is not None else None, ctypes.byref(ticket), self._stream()))
        return int(ticket.value)

    def host_wait(self, ticket: int):
        """(loss, dt_prime, dbias) of a submitted step, as Python floats, once they are on the host."""
        out = (ctypes.c_float * 3)()
        p = ctypes.cast(out, ctypes.c_void_p).value
        _capi.check(self._L.siglip_host_wait(self._h, ticket, p, p + 4, p + 8))
        return float(out[0]), float(out[1]), float(out[2])

    def _check_host(self, img_host: torch.Tensor, txt_host: torch.Tensor) -> None:
        for x in (img_host, txt_host):
            if x.device.type != "cpu" or x.dtype != torch.bfloat16 or not x.is_contiguous() or \
                    tuple(x.shape) != (self.batch, self.dim):
                raise RuntimeError("the host entries expect contiguous CPU bf16 tensors of shape [B, D]")

    def _check(self, img: torch.Tensor, txt: torch.Tensor) -> None:
        """Operands are contiguous device tensors, img [R, D] and txt [T, D] (R = T = B without extras), both bf16
        (default format) or both float16 holding 16*x (the fp32-input format, see convert_f32); the context option
        follows the dtype."""
        for x, n in ((img, self.images), (txt, self.texts)):
            if x.device != self.device or x.dtype not in (torch.bfloat16, torch.float16) or not x.is_contiguous() or \
                    tuple(x.shape) != (n, self.dim):
                raise RuntimeError(
                    f"expected contiguous bf16 (or fp16 x16) [{n}, {self.dim}] tensors on {self.device}, got "
                    f"{tuple(x.shape)} {x.dtype} on {x.device}")
        if img.dtype != txt.dtype:
            raise RuntimeError("image and text operands must use the same 16-bit format")
        self._set_input_f16(img.dtype == torch.float16)

    def _set_tprime_f64(self, t_prime: torch.Tensor) -> bool:
        """t' may be handed over as the reference holds it (fp64, distributed_sigmoid_loss.py:11) or as fp32; dt' then
        comes back in the same dtype. The context option follows the tensor."""
        if t_prime.dtype not in (torch.float32, torch.float64) or t_prime.numel() != 1 or t_prime.device != self.device:
            raise RuntimeError("t_prime must be a 1-element fp32 or fp64 tensor on the engine's device")
        f64 = t_prime.dtype == torch.float64
        if f64 != getattr(self, "_tprime_f64", False):
            _capi.check(self._L.siglip_ctx_set_option(self._h, _capi.SIGLIP_OPT_TPRIME_F64, int(f64)))
            self._tprime_f64 = f64
        return f64

    def _set_input_f16(self, f16: bool) -> None:
        if f16 != getattr(self, "_input_f16", False):
            _capi.check(self._L.siglip_ctx_set_option(self._h, _capi.SIGLIP_OPT_INPUT_F16, int(f16)))
            self._input_f16 = f16

    def convert_f32(self, x: torch.Tensor, f16: bool) -> torch.Tensor:
        """The module's cast of fp32 embeddings to the kernels' operand format: bf16 (f16=False, == x.to(bfloat16)) or
        float16 holding 16*x (f16=True: 11 significant bits, what fp32 callers get)."""
        if not self._rows_ok(x) or x.dtype != torch.float32 or not x.is_contiguous() or x.device != self.device:
            raise RuntimeError(f"convert_f32 expects a contiguous fp32 [{self.batch}, {self.texts} or {self.images}, "
                               f"{self.dim}] tensor "
                               f"on {self.device}")
        self._set_input_f16(f16)
        out = torch.empty(x.shape[0], self.dim, device=self.device, dtype=torch.float16 if f16 else torch.bfloat16)
        with torch.cuda.device(self.device):
            _capi.check(self._L.siglip_convert_f32_rows(self._h, x.shape[0], x.data_ptr(), out.data_ptr(),
                                                        self._stream()))
        return out

    def close(self) -> None:
        if getattr(self, "_h", None) is not None and self._h.value:
            self._L.siglip_ctx_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):  # best effort
        try:
            self.close()
        except Exception:
            pass


def _aligned(x: torch.Tensor) -> torch.Tensor:
    """Contiguous and 16-byte aligned (TMA / 16-byte vector accesses): a view into the middle of a storage is cloned
    instead of rejected."""
    x = x.contiguous()
    return x if x.data_ptr() % 16 == 0 else x.clone()


class _SigmoidLossFn(torch.autograd.Function):
    """loss = sum_chunks(-logsigmoid(labels * (img @ txt_chunk.T * exp(t') + b))).sum() / B.

    Two schedules, same kernels, same results (SURVEY.md §0: the four gradients depend on the logits and ONE upstream
    scalar only):
      * split  (fused=False): forward = the W loss kernels, the sigma operands of all W chunks stay in the engine;
        backward = the W gradient kernels with grad_output folded into their epilogues. O(W B^2) workspace.
      * fused  (fused=True): forward = the fused step (loss and gradient kernels alternating chunk by chunk, two sigma
        operands, every cross-rank flag handled inside the kernels) which leaves the gradients for an upstream gradient
        of 1; backward = one multiply by grad_output per tensor (siglip_scale). O(B^2) workspace.
    normalize=True additionally fuses F.normalize of both inputs (forward) and its backward around the loss.
    ids: [B] int64 sample ids (SIGLIP_OPT_SAMPLE_IDS engines), set before every step the engine runs for this call.
    extra_ids: [T - B] int64 ids of the extra texts (SIGLIP_OPT_EXTRA_TEXT_IDS engines), set along with ids.
    metrics: (top1, i2t_index, t2i_index) output buffers: the retrieval metrics of this call's step are armed. A re-run
    of the forward by the backward's generation guard does not arm them again (they belong to the first run).
    weights: (image_weights [R] or None, text_weights [T] or None) fp32 (SIGLIP_OPT_SAMPLE_WEIGHTS engines), set before
    every step the engine runs for this call, like the ids.
    extra_img_ids: [R - B] int64 ids of the extra images (SIGLIP_OPT_EXTRA_IMAGE_IDS engines), set along with ids.
    teacher: (teacher_image, teacher_text, teacher_t_prime, teacher_bias, lambda) of a distillation step
    (SIGLIP_OPT_DISTILL engines): constants, no gradient flows to them; set before every step like the ids.
    sample_losses: (image_loss [R], text_loss [T]) fp32 output buffers: the per-sample losses of this call's step are
    armed. Like the metrics, a re-run of the forward by the backward's generation guard does not arm them again.
    groups: (image_groups [R], text_groups [T]) int64 (SIGLIP_OPT_EXCLUDE_GROUPS engines), set before every step the
    engine runs for this call, like the ids.
    label_sets: (sample_labels [B, M], extra_text_labels [T - B, M] or None, extra_image_labels [R - B, M] or None) int64
    (SIGLIP_OPT_LABEL_SETS engines), set before every step the engine runs for this call, like the ids."""

    @staticmethod
    def forward(ctx, img, txt, t_prime, bias, engine: SigmoidLossEngine, normalize: bool = False, fused: bool = False,
                ids: Optional[torch.Tensor] = None, metrics=None, extra_ids: Optional[torch.Tensor] = None, weights=None,
                extra_img_ids: Optional[torch.Tensor] = None, teacher=None, sample_losses=None, groups=None,
                label_sets=None):
        need_grad = any(ctx.needs_input_grad[:4])
        raw = None
        # bf16 callers: bf16 operands (what autograd would multiply). Anything wider (the reference's own test feeds
        # fp32): fp16 operands holding 16*x — 11 significant bits instead of 8 (gradient error vs the fp32 reference
        # 2e-4 instead of 1.7e-3)
        hi = not (img.dtype == torch.bfloat16 and txt.dtype == torch.bfloat16)
        if normalize:
            def prep(x):
                x = x.detach()
                if x.dtype not in (torch.float32, torch.bfloat16):
                    x = x.float()
                return _aligned(x)
            img_r, txt_r = prep(img), prep(txt)
            img_b, inv_i = engine.normalize_fwd(img_r, hi)
            txt_b, inv_t = engine.normalize_fwd(txt_r, hi)
            raw = (img_r, txt_r, inv_i, inv_t)
        elif hi:
            img_b = engine.convert_f32(_aligned(img.detach().float()), True)
            txt_b = engine.convert_f32(_aligned(txt.detach().float()), True)
        else:
            img_b = _aligned(img.detach())
            txt_b = _aligned(txt.detach())
        # the two scalars go to the kernels as the module holds them (t' fp64 like the reference's parameter, bias
        # fp32): no conversion kernels in the stream; anything else is converted to fp32 first
        tp = t_prime.detach()
        if not (tp.device == img.device and tp.dtype in (torch.float32, torch.float64)):
            tp = tp.to(device=img.device, dtype=torch.float32)
        tp = tp.reshape(1)
        b = bias.detach()
        if not (b.device == img.device and b.dtype == torch.float32):
            b = b.to(device=img.device, dtype=torch.float32)
        b = b.reshape(1)
        ctx.fused = bool(fused and need_grad)
        if teacher is not None:
            timg, ttxt, ttp, tbias, lam = teacher
            teacher = (engine.teacher_operand(timg.detach(), normalize), engine.teacher_operand(ttxt.detach(), normalize),
                       ttp.detach().to(device=img.device, dtype=torch.float32).reshape(1),
                       tbias.detach().to(device=img.device, dtype=torch.float32).reshape(1), lam)
            engine.set_teacher(*teacher)
        ctx.ids, ctx.extra_ids, ctx.weights, ctx.extra_img_ids = ids, extra_ids, weights, extra_img_ids
        ctx.groups = groups
        ctx.label_sets = label_sets
        # the split schedule's backward may have to re-run the forward with the same teacher; the fused one never does
        ctx.teacher = None if ctx.fused else teacher
        if ids is not None:
            engine.set_sample_ids(ids)
        if extra_ids is not None:
            engine.set_extra_text_ids(extra_ids)
        if extra_img_ids is not None:
            engine.set_extra_image_ids(extra_img_ids)
        if weights is not None:
            engine.set_sample_weights(*weights)
        if groups is not None:
            engine.set_groups(*groups)
        if label_sets is not None:
            engine.set_label_sets(*label_sets)
        if metrics is not None:
            engine.request_metrics(*metrics[:3])
            if len(metrics) > 3:   # metrics_topk = K > 1: (K, recall, i2t_topk, t2i_topk) follow
                engine.request_topk(*metrics[3:])
        if sample_losses is not None:
            engine.request_sample_losses(*sample_losses)
        if ctx.fused:
            # gradients in the dtype autograd would return for these inputs (fp32 when a projection follows)
            gdt = torch.bfloat16 if (not hi and not normalize) else torch.float32
            loss, dimg, dtxt, dtp, db = engine.fwd_bwd(img_b, txt_b, tp, b, gdt)
            saved = [dimg, dtxt, dtp, db]
            if raw is not None:
                saved += list(raw)
            ctx.save_for_backward(*saved)
        else:
            loss = engine.forward(img_b, txt_b, tp, b, need_grad)
            if need_grad:
                if raw is not None:
                    ctx.save_for_backward(img_b, txt_b, tp, b, *raw)
                else:
                    ctx.save_for_backward(img_b, txt_b, tp, b)
                ctx.gen = engine.saved_generation
        if need_grad:
            ctx.normalize = normalize
            ctx.engine = engine
            ctx.in_meta = (img.dtype, txt.dtype, t_prime.dtype, bias.dtype, t_prime.shape, bias.shape,
                           t_prime.device, bias.device)
        # reference result dtype: promote(input dtype, fp32 labels) (distributed_sigmoid_loss.py:28-32)
        out_dtype = torch.promote_types(img.dtype, torch.float32)
        return loss.reshape(()).to(out_dtype)

    @staticmethod
    def backward(ctx, grad_out):
        saved = ctx.saved_tensors
        eng = ctx.engine
        idt, tdt, pdt, bdt, pshape, bshape, pdev, bdev = ctx.in_meta
        g = grad_out.detach().to(torch.float32).reshape(1).contiguous()
        if ctx.fused:
            dimg, dtxt, dtp, db = saved[:4]
            if ctx.normalize:
                img_r, txt_r, inv_i, inv_t = saved[4:]
                gi = eng.normalize_bwd(img_r, inv_i, eng.scale(dimg, g)).to(idt) if ctx.needs_input_grad[0] else None
                gt = eng.normalize_bwd(txt_r, inv_t, eng.scale(dtxt, g)).to(tdt) if ctx.needs_input_grad[1] else None
            else:
                gi = eng.scale(dimg, g).to(idt) if ctx.needs_input_grad[0] else None
                gt = eng.scale(dtxt, g).to(tdt) if ctx.needs_input_grad[1] else None
            sc = eng.scale(torch.cat([dtp.float(), db]), g)
            dtp, db = sc[0:1], sc[1:2]
        else:
            img_b, txt_b, tp, b = saved[:4]
            if eng.saved_generation != ctx.gen:
                # another forward of the same module ran in between: rebuild the saved state (every rank takes this
                # branch together, so the collective stays matched); the re-run takes this call's ids and weights again
                if ctx.ids is not None:
                    eng.set_sample_ids(ctx.ids)
                if ctx.extra_ids is not None:
                    eng.set_extra_text_ids(ctx.extra_ids)
                if ctx.extra_img_ids is not None:
                    eng.set_extra_image_ids(ctx.extra_img_ids)
                if ctx.weights is not None:
                    eng.set_sample_weights(*ctx.weights)
                if ctx.groups is not None:
                    eng.set_groups(*ctx.groups)
                if ctx.label_sets is not None:
                    eng.set_label_sets(*ctx.label_sets)
                if ctx.teacher is not None:
                    eng.set_teacher(*ctx.teacher)
                eng.forward(img_b, txt_b, tp, b, True)
                ctx.gen = eng.saved_generation
            if ctx.normalize:
                # fp32 gradients w.r.t. the normalised embeddings, then the projection of F.normalize's backward
                img_r, txt_r, inv_i, inv_t = saved[4:]
                dimg, dtxt, dtp, db = eng.backward(img_b, txt_b, tp, g, torch.float32)
                gi = eng.normalize_bwd(img_r, inv_i, dimg).to(idt) if ctx.needs_input_grad[0] else None
                gt = eng.normalize_bwd(txt_r, inv_t, dtxt).to(tdt) if ctx.needs_input_grad[1] else None
            else:
                # gradients in the dtype autograd would return for these inputs: bf16 straight from the kernel epilogue
                gdt = torch.bfloat16 if (idt == torch.bfloat16 and tdt == torch.bfloat16) else torch.float32
                dimg, dtxt, dtp, db = eng.backward(img_b, txt_b, tp, g, gdt)
                gi = dimg.to(idt) if ctx.needs_input_grad[0] else None
                gt = dtxt.to(tdt) if ctx.needs_input_grad[1] else None
        gp = dtp.reshape(pshape).to(device=pdev, dtype=pdt) if ctx.needs_input_grad[2] else None
        gb = db.reshape(bshape).to(device=bdev, dtype=bdt) if ctx.needs_input_grad[3] else None
        return gi, gt, gp, gb, None, None, None, None, None, None, None, None, None, None, None, None


class _EngineCache:
    def __init__(self, group=None, cta_group: int = 2, overlap_pull: bool = True, sync_scalar_grads: bool = False,
                 bidir: bool = False, batch_per_rank=None, multi_positive: bool = False, hard_negatives: int = 0,
                 extra_texts: int = 0, sample_weights: bool = False, extra_images: int = 0,
                 distill: Optional[float] = None, sigma_budget_bytes: Optional[int] = None,
                 exclude_groups: bool = False, multi_label: int = 0, focal=None, distill_options: bool = False):
        self.group, self.cta_group, self.overlap_pull = group, cta_group, overlap_pull
        self.distill_options = distill_options
        self.focal = focal   # (gamma, alpha or None), or None
        self.exclude_groups = exclude_groups
        self.multi_label = multi_label
        self.sigma_budget_bytes = sigma_budget_bytes
        self.distill = distill
        self.extra_images = extra_images
        self.sample_weights = sample_weights
        self.sync_scalar_grads, self.bidir = sync_scalar_grads, bidir
        self.multi_positive = multi_positive
        self.batch_per_rank = batch_per_rank
        self.hard_negatives = hard_negatives
        self.extra_texts = extra_texts
        self._engines: Dict[Tuple[int, int, int, int], SigmoidLossEngine] = {}

    def get(self, batch: int, dim: int, device: torch.device, teacher_dim: int = 0) -> SigmoidLossEngine:
        key = (device.index if device.index is not None else torch.cuda.current_device(), batch, dim, teacher_dim)
        eng = self._engines.get(key)
        if eng is None:
            dev = torch.device("cuda", key[0])
            tpr = ipr = None
            extras = self.hard_negatives + self.extra_texts   # at most one of the two is non-zero
            rank, world = _group_rank_world(self.group)
            bpr = self.batch_per_rank if self.batch_per_rank is not None else [batch] * world
            if extras:
                # every rank scores the same number K of extras: T_p = B_p + K
                tpr = [int(b) + extras for b in bpr]
            if self.extra_images:
                # every rank holds the same number K of extra images: R_p = B_p + K
                ipr = [int(b) + self.extra_images for b in bpr]
            eng = SigmoidLossEngine(batch, dim, dev, self.group, self.cta_group, self.overlap_pull,
                                    batch_per_rank=self.batch_per_rank, texts_per_rank=tpr, images_per_rank=ipr,
                                    teacher_dim=teacher_dim, labels=self.multi_label,
                                    distill_options=self.distill_options and teacher_dim > 0)
            if self.sync_scalar_grads:
                eng.set_option(_capi.SIGLIP_OPT_SYNC_SCALAR_GRADS, 1)
            if self.bidir:
                eng.set_option(_capi.SIGLIP_OPT_BIDIR, 1)
            if self.multi_positive:
                eng.set_option(_capi.SIGLIP_OPT_SAMPLE_IDS, 1)
            if self.multi_label:
                eng.set_option(_capi.SIGLIP_OPT_LABEL_SETS, 1)
            if self.extra_texts and not self.multi_label:
                eng.set_option(_capi.SIGLIP_OPT_EXTRA_TEXT_IDS, 1)   # needs the sample ids on first
            if self.extra_images and self.multi_positive:
                eng.set_option(_capi.SIGLIP_OPT_EXTRA_IMAGE_IDS, 1)
            if self.sample_weights:
                eng.set_option(_capi.SIGLIP_OPT_SAMPLE_WEIGHTS, 1)
            if self.distill is not None:
                eng.set_option(_capi.SIGLIP_OPT_DISTILL, 1)
            if self.exclude_groups:
                eng.set_option(_capi.SIGLIP_OPT_EXCLUDE_GROUPS, 1)
            if self.focal is not None:
                eng.set_option(_capi.SIGLIP_OPT_FOCAL, 1)
                eng.set_focal(*self.focal)
            if self.sigma_budget_bytes:
                eng.set_sigma_budget(self.sigma_budget_bytes)
            self._engines[key] = eng
        return eng


def _sigma_budget_mib(sigma_budget_bytes) -> int:
    if sigma_budget_bytes is None:
        return 0
    if isinstance(sigma_budget_bytes, bool) or not isinstance(sigma_budget_bytes, int) or sigma_budget_bytes < 0:
        raise ValueError(f"sigma_budget_bytes must be None or an int >= 0, got {sigma_budget_bytes!r}")
    mib = sigma_budget_bytes >> 20
    if sigma_budget_bytes and mib == 0:
        raise ValueError(f"sigma_budget_bytes = {sigma_budget_bytes} is below 1 MiB")
    return mib


def _fused_under_budget(eng, fused_step: Optional[bool]) -> bool:
    """The schedule of a step: the module's choice, except that under a sigma budget every step takes the fused step
    (the split forward keeps W whole operands); an explicit fused_step=False that the budget cannot hold raises here,
    before any GPU work."""
    fused = (eng.world > 1) if fused_step is None else bool(fused_step)
    if getattr(eng, "sigma_budget_mib", 0):
        if fused_step is None:
            fused = True
        elif not fused and not eng.split_fits_budget():
            raise ValueError("fused_step=False keeps one whole sigma operand per rank until the backward, more than "
                             "sigma_budget_bytes: use fused_step=None or True, which runs in row panels")
    return fused


_ID_DTYPES = (torch.int8, torch.uint8, torch.int16, torch.int32, torch.int64)


def _validate_ids(sample_ids, multi_positive: bool, embeddings: torch.Tensor) -> Optional[torch.Tensor]:
    """sample_ids of a forward: required ([B] integers on the embeddings' device) with multi_positive, refused without.
    Returns them as contiguous int64 (what the kernels compare), or None. Raises before any GPU work."""
    if not multi_positive:
        if sample_ids is not None:
            raise RuntimeError("sample_ids given, but the loss was built without multi_positive=True")
        return None
    if sample_ids is None:
        raise RuntimeError("multi_positive=True: forward needs sample_ids ([batch] integer tensor, one id per sample)")
    if not isinstance(sample_ids, torch.Tensor) or sample_ids.dtype not in _ID_DTYPES:
        raise RuntimeError(f"sample_ids must be an integer tensor, got "
                           f"{sample_ids.dtype if isinstance(sample_ids, torch.Tensor) else type(sample_ids)}")
    batch = embeddings.shape[0] if embeddings.dim() >= 1 else None
    if sample_ids.dim() != 1 or sample_ids.shape[0] != batch:
        raise RuntimeError(f"sample_ids must have shape [{batch}] (one id per sample), got {tuple(sample_ids.shape)}")
    if sample_ids.device != embeddings.device:
        raise RuntimeError(f"sample_ids are on {sample_ids.device}, the embeddings on {embeddings.device}")
    return sample_ids.to(torch.int64).contiguous()


def _validate_hard_negatives(hard_negatives, name: str = "hard_negatives") -> int:
    if isinstance(hard_negatives, bool) or not isinstance(hard_negatives, int) or hard_negatives < 0:
        raise RuntimeError(f"{name} must be an int >= 0, got {hard_negatives!r}")
    return hard_negatives


def _validate_extra_texts(extra_texts, multi_positive: bool, hard_negatives: int) -> int:
    """extra_texts=K of a module: K extra captions per rank with ids of their own, so it needs the sample ids of
    multi_positive, and it is a different meaning of the extras than hard_negatives (never positive)."""
    extra_texts = _validate_hard_negatives(extra_texts, "extra_texts")
    if extra_texts and not multi_positive:
        raise RuntimeError("extra_texts=K needs multi_positive=True (the extras' ids are compared with the sample ids)")
    if extra_texts and hard_negatives:
        raise RuntimeError("extra_texts and hard_negatives cannot be combined: give the hard negatives as extra texts "
                           "whose ids match no image")
    return extra_texts


def _validate_negatives(text_embeddings: torch.Tensor, negative_text, hard_negatives: int,
                        name: str = "negative_text", option: str = "hard_negatives", what: str = "texts") -> None:
    """negative_text of a forward: required ([K, D], the dtype / device / width of the texts) when the loss was built
    with hard_negatives = K > 0, refused otherwise. Raises before any GPU work. (name / option / what: the same check for
    extra_text and extra_texts, and for extra_image and extra_images against the images.)"""
    if hard_negatives == 0:
        if negative_text is not None:
            raise RuntimeError(f"{name} given, but the loss was built without {option} ({option}=K)")
        return
    if negative_text is None:
        raise RuntimeError(f"{option}={hard_negatives}: forward needs {name} ([{hard_negatives}, emb_dim])")
    if not isinstance(negative_text, torch.Tensor):
        raise RuntimeError(f"{name} must be a tensor, got {type(negative_text).__name__}")
    want = (hard_negatives, text_embeddings.shape[1] if text_embeddings.dim() == 2 else None)
    if negative_text.dim() != 2 or tuple(negative_text.shape) != want:
        raise RuntimeError(f"{name} must have shape [{want[0]}, {want[1]}] ({option} x the {what}' width), "
                           f"got {tuple(negative_text.shape)}")
    if negative_text.dtype != text_embeddings.dtype:
        raise RuntimeError(f"{name} is {negative_text.dtype}, the {what} {text_embeddings.dtype}")
    if negative_text.device != text_embeddings.device:
        raise RuntimeError(f"{name} is on {negative_text.device}, the {what} on {text_embeddings.device}")


def _validate_extra_text_ids(extra_text_ids, extra_texts: int, text_embeddings: torch.Tensor) -> Optional[torch.Tensor]:
    """extra_text_ids of a forward: required ([K] integers on the texts' device) when the loss was built with
    extra_texts = K > 0, refused otherwise. Returns them as contiguous int64, or None. Raises before any GPU work."""
    if extra_texts == 0:
        if extra_text_ids is not None:
            raise RuntimeError("extra_text_ids given, but the loss was built without extra_texts (extra_texts=K)")
        return None
    if extra_text_ids is None:
        raise RuntimeError(f"extra_texts={extra_texts}: forward needs extra_text_ids ([{extra_texts}] integer tensor)")
    if not isinstance(extra_text_ids, torch.Tensor) or extra_text_ids.dtype not in _ID_DTYPES:
        raise RuntimeError(f"extra_text_ids must be an integer tensor, got "
                           f"{extra_text_ids.dtype if isinstance(extra_text_ids, torch.Tensor) else type(extra_text_ids)}")
    if extra_text_ids.dim() != 1 or extra_text_ids.shape[0] != extra_texts:
        raise RuntimeError(f"extra_text_ids must have shape [{extra_texts}] (one id per extra text), got "
                           f"{tuple(extra_text_ids.shape)}")
    if extra_text_ids.device != text_embeddings.device:
        raise RuntimeError(f"extra_text_ids are on {extra_text_ids.device}, the texts on {text_embeddings.device}")
    return extra_text_ids.to(torch.int64).contiguous()


def _validate_extra_image_ids(extra_image_ids, extra_images: int, multi_positive: bool,
                              image_embeddings: torch.Tensor) -> Optional[torch.Tensor]:
    """extra_image_ids of a forward: required ([K] integers on the images' device) when the loss was built with
    extra_images = K > 0 and multi_positive=True (several images per caption), refused otherwise (without ids the extra
    images are hard negatives). Returns them as contiguous int64, or None. Raises before any GPU work."""
    if extra_images == 0 or not multi_positive:
        if extra_image_ids is not None:
            raise RuntimeError("extra_image_ids given, but the loss was built without extra_images=K and "
                               "multi_positive=True (without ids the extra images are hard negatives)")
        return None
    if extra_image_ids is None:
        raise RuntimeError(f"extra_images={extra_images} with multi_positive=True: forward needs extra_image_ids "
                           f"([{extra_images}] integer tensor)")
    if not isinstance(extra_image_ids, torch.Tensor) or extra_image_ids.dtype not in _ID_DTYPES:
        raise RuntimeError(f"extra_image_ids must be an integer tensor, got "
                           f"{extra_image_ids.dtype if isinstance(extra_image_ids, torch.Tensor) else type(extra_image_ids)}")
    if extra_image_ids.dim() != 1 or extra_image_ids.shape[0] != extra_images:
        raise RuntimeError(f"extra_image_ids must have shape [{extra_images}] (one id per extra image), got "
                           f"{tuple(extra_image_ids.shape)}")
    if extra_image_ids.device != image_embeddings.device:
        raise RuntimeError(f"extra_image_ids are on {extra_image_ids.device}, the images on {image_embeddings.device}")
    return extra_image_ids.to(torch.int64).contiguous()


def _validate_sample_weights(sample_weights) -> bool:
    if not isinstance(sample_weights, bool):
        raise RuntimeError(f"sample_weights must be a bool, got {type(sample_weights).__name__}")
    return sample_weights


def _validate_weights(weights, sample_weights: bool, n: Optional[int], name: str,
                      device: torch.device) -> Optional[torch.Tensor]:
    """image_weights / text_weights of a forward: accepted only when the loss was built with sample_weights=True. None
    means ones; otherwise a floating [n] tensor on the embeddings' device that does not require grad (the weights are
    inputs: no gradient with respect to them is computed). Returns it as contiguous fp32, or None. Raises before any GPU
    work. Values outside [0, 1] are clamped into it by the copy (NaN -> 0)."""
    if not sample_weights:
        if weights is not None:
            raise RuntimeError(f"{name} given, but the loss was built without sample_weights=True")
        return None
    if weights is None:
        return None
    if not isinstance(weights, torch.Tensor) or not weights.is_floating_point():
        raise RuntimeError(f"{name} must be a floating-point tensor, got "
                           f"{weights.dtype if isinstance(weights, torch.Tensor) else type(weights).__name__}")
    if weights.dim() != 1 or weights.shape[0] != n:
        raise RuntimeError(f"{name} must have shape [{n}], got {tuple(weights.shape)}")
    if weights.device != device:
        raise RuntimeError(f"{name} is on {weights.device}, the embeddings on {device}")
    if weights.requires_grad:
        raise RuntimeError(f"{name} requires grad, but no gradient with respect to the sample weights is computed: "
                           f"pass {name}.detach()")
    return weights.to(torch.float32).contiguous()


def _weights_of(sample_weights: bool, image_weights, text_weights, image_embeddings: torch.Tensor,
                text_embeddings: torch.Tensor, extras: int, extra_images: int = 0):
    """Both weight arguments checked; (image_weights, text_weights) for the step, or None without sample_weights. The
    texts are the paired ones followed by the K extras, so text_weights has B + K entries; the images likewise, so
    image_weights has B + K_img entries."""
    rows = lambda x: x.shape[0] if x.dim() >= 1 else None  # noqa: E731
    ni = rows(image_embeddings)
    iw = _validate_weights(image_weights, sample_weights, ni + extra_images if ni is not None else None,
                           "image_weights", image_embeddings.device)
    nt = rows(text_embeddings)
    tw = _validate_weights(text_weights, sample_weights, nt + extras if nt is not None else None, "text_weights",
                           text_embeddings.device)
    return (iw, tw) if sample_weights else None


def _validate_exclude_groups(exclude_groups, distill) -> bool:
    """exclude_groups of a module: a bool, and not together with distill unless distill_options=True (distill: the
    module's distill_closed)."""
    if not isinstance(exclude_groups, bool):
        raise RuntimeError(f"exclude_groups must be a bool, got {type(exclude_groups).__name__}")
    if exclude_groups and distill is not None:
        raise RuntimeError("exclude_groups cannot be combined with distill: the distillation loss kernel does not "
                           "exclude pairs (distill_options=True runs the one that does)")
    return exclude_groups


def _validate_group_ids(groups, n: Optional[int], name: str, what: str, device: torch.device) -> torch.Tensor:
    if groups is None:
        raise RuntimeError(f"exclude_groups=True: forward needs {name} ([{n}] integer tensor, one group per {what[:-1]})")
    if not isinstance(groups, torch.Tensor) or groups.dtype not in _ID_DTYPES:
        raise RuntimeError(f"{name} must be an integer tensor, got "
                           f"{groups.dtype if isinstance(groups, torch.Tensor) else type(groups)}")
    if groups.dim() != 1 or groups.shape[0] != n:
        raise RuntimeError(f"{name} must have shape [{n}] (one group per {what[:-1]}), got {tuple(groups.shape)}")
    if groups.device != device:
        raise RuntimeError(f"{name} are on {groups.device}, the {what} on {device}")
    return groups.to(torch.int64).contiguous()


def _groups_of(exclude_groups: bool, image_groups, text_groups, image_embeddings: torch.Tensor,
               text_embeddings: torch.Tensor, extras: int, extra_images: int):
    """image_groups / text_groups of a forward: both required with exclude_groups, refused without. The images are the
    paired ones followed by the extra images ([B + K_img]), the texts the paired ones followed by the hard negatives or
    extra texts ([B + K]). Returns them as contiguous int64, or None. Raises before any GPU work."""
    if not exclude_groups:
        for name, v in (("image_groups", image_groups), ("text_groups", text_groups)):
            if v is not None:
                raise RuntimeError(f"{name} given, but the loss was built without exclude_groups=True")
        return None
    ni = image_embeddings.shape[0] if image_embeddings.dim() >= 1 else None
    nt = text_embeddings.shape[0] if text_embeddings.dim() >= 1 else None
    gi = _validate_group_ids(image_groups, ni + extra_images if ni is not None else None, "image_groups", "images",
                             image_embeddings.device)
    gt = _validate_group_ids(text_groups, nt + extras if nt is not None else None, "text_groups", "texts",
                             text_embeddings.device)
    return gi, gt


def _validate_multi_label(multi_label, multi_positive: bool, distill) -> int:
    """multi_label=M of a module: None or 0 (off), or the labels per set, 1 .. MAX_LABELS. Label sets replace the ids of
    multi_positive, and need distill_options=True under distill (distill: the module's distill_closed)."""
    if multi_label is None:
        return 0
    if isinstance(multi_label, bool) or not isinstance(multi_label, int) or not 0 <= multi_label <= MAX_LABELS:
        raise RuntimeError(f"multi_label must be None or an int in 1 .. {MAX_LABELS} (labels per set), got "
                           f"{multi_label!r}")
    if multi_label and multi_positive:
        raise RuntimeError("multi_label cannot be combined with multi_positive: label sets replace the sample ids "
                           "(M = 1 with the ids as labels is multi_positive)")
    if multi_label and distill is not None:
        raise RuntimeError("multi_label cannot be combined with distill: the distillation loss kernel has no label sets "
                           "(distill_options=True runs the one that has)")
    return multi_label


def _validate_label_set(labels, n: Optional[int], m: int, name: str, what: str, device: torch.device) -> torch.Tensor:
    if labels is None:
        raise RuntimeError(f"multi_label={m}: forward needs {name} ([{n}, {m}] integer tensor, one label set per "
                           f"{what})")
    if not isinstance(labels, torch.Tensor) or labels.dtype not in _ID_DTYPES:
        raise RuntimeError(f"{name} must be an integer tensor, got "
                           f"{labels.dtype if isinstance(labels, torch.Tensor) else type(labels)}")
    if labels.dim() != 2 or tuple(labels.shape) != (n, m):
        raise RuntimeError(f"{name} must have shape [{n}, {m}] (one set of {m} labels per {what}), got "
                           f"{tuple(labels.shape)}")
    if labels.device != device:
        raise RuntimeError(f"{name} are on {labels.device}, the embeddings on {device}")
    return labels.to(torch.int64).contiguous()


def _label_sets_of(multi_label: int, sample_labels, extra_text_labels, extra_image_labels,
                   image_embeddings: torch.Tensor, extra_texts: int, extra_images: int):
    """sample_labels [B, M] / extra_text_labels [K, M] / extra_image_labels [K_img, M] of a forward: the sample sets are
    required with multi_label, the extra texts' with extra_texts = K > 0 and the extra images' with extra_images =
    K_img > 0; every one is refused otherwise (hard negatives get empty sets). A negative label is an empty slot.
    Returns (sample, extra text or None, extra image or None) as contiguous int64, or None. Raises before any GPU
    work."""
    given = (("sample_labels", sample_labels), ("extra_text_labels", extra_text_labels),
             ("extra_image_labels", extra_image_labels))
    if not multi_label:
        for name, v in given:
            if v is not None:
                raise RuntimeError(f"{name} given, but the loss was built without multi_label=M")
        return None
    if extra_texts == 0 and extra_text_labels is not None:
        raise RuntimeError("extra_text_labels given, but the loss was built without extra_texts=K (hard negatives have "
                           "empty label sets)")
    if extra_images == 0 and extra_image_labels is not None:
        raise RuntimeError("extra_image_labels given, but the loss was built without extra_images=K")
    dev = image_embeddings.device
    nb = image_embeddings.shape[0] if image_embeddings.dim() >= 1 else None
    ls = _validate_label_set(sample_labels, nb, multi_label, "sample_labels", "sample", dev)
    lt = _validate_label_set(extra_text_labels, extra_texts, multi_label, "extra_text_labels", "extra text",
                             dev) if extra_texts else None
    li = _validate_label_set(extra_image_labels, extra_images, multi_label, "extra_image_labels", "extra image",
                             dev) if extra_images else None
    return ls, lt, li


def _with_negatives(text_embeddings: torch.Tensor, negative_text) -> torch.Tensor:
    """[txt; negative_text] as one contiguous operand; torch.cat is differentiable, so negative_text.grad comes back
    through autograd."""
    return text_embeddings if negative_text is None else torch.cat([text_embeddings, negative_text])


def _validate_focal(focal_gamma, focal_alpha, distill):
    """focal_gamma / focal_alpha of a module: None (off), or gamma a finite number in [0, 8] and alpha None or a number
    in [0, 1]. |g| < 1.44 for gamma <= 8 keeps every pair derivative inside the fp16 sigma operand. Not with distill:
    the distillation loss kernel has no focal terms. Returns (gamma, alpha) or None."""
    def number(x):
        return not isinstance(x, bool) and isinstance(x, (int, float))
    if focal_gamma is None:
        if focal_alpha is not None:
            raise RuntimeError("focal_alpha given, but the loss was built without focal_gamma")
        return None
    if not number(focal_gamma) or not 0.0 <= float(focal_gamma) <= 8.0:   # NaN fails the comparison
        raise RuntimeError(f"focal_gamma must be None or a number in [0, 8], got {focal_gamma!r}")
    if focal_alpha is not None and (not number(focal_alpha) or not 0.0 <= float(focal_alpha) <= 1.0):
        raise RuntimeError(f"focal_alpha must be None or a number in [0, 1], got {focal_alpha!r}")
    if distill is not None:
        raise RuntimeError("focal_gamma cannot be combined with distill: the distillation loss kernel has no focal terms")
    return float(focal_gamma), (None if focal_alpha is None else float(focal_alpha))


def _validate_distill(distill, hard_negatives: int, extra_texts: int, extra_images: int,
                      distill_options=False) -> Optional[float]:
    """distill=lambda of a module: None (off) or a float in (0, 1], the weight of the teacher's probabilities in the
    targets. The extras of hard_negatives / extra_texts / extra_images need teacher embeddings of their own, which
    only distill_options=True takes (a bool, and only with distill)."""
    if not isinstance(distill_options, bool):
        raise RuntimeError(f"distill_options must be a bool, got {type(distill_options).__name__}")
    if distill_options and distill is None:
        raise RuntimeError("distill_options=True needs distill=lambda")
    if distill is None:
        return None
    if isinstance(distill, bool) or not isinstance(distill, (int, float)) or not 0.0 < float(distill) <= 1.0:
        raise RuntimeError(f"distill must be a float in (0, 1] (the weight of the teacher's probabilities), got "
                           f"{distill!r}")
    for name, k in (("hard_negatives", hard_negatives), ("extra_texts", extra_texts), ("extra_images", extra_images)):
        if k and not distill_options:
            raise RuntimeError(f"distill cannot be combined with {name}: its extra embeddings would need teacher "
                               f"embeddings of their own (distill_options=True takes them)")
    return float(distill)


def _teacher_of(distill: Optional[float], image_embeddings: torch.Tensor, names, values, extras=()):
    """The teacher arguments of a forward: all four required with distill, refused without. teacher_image and
    teacher_text are floating [B, D_T] tensors (the same shape, D_T may differ from the students' width) and the two
    scalars 1-element floating tensors, all on the embeddings' device, none requiring grad: the teacher is a constant
    and a gradient with respect to it is never computed. extras: (name, tensor, K, "text" or "image") of the teacher's
    rows for the student's extras (teacher_negative_text, teacher_extra_text, teacher_extra_image): each required
    exactly when its K > 0, a [K, D_T] tensor checked like the others and of its paired tensor's dtype, appended to
    teacher_text or teacher_image in the student's order. Returns (timg, ttxt, scale, bias, lambda) with D_T
    zero-padded to a multiple of 8, or None. Raises before any GPU work."""
    if distill is None:
        for n, x in list(zip(names, values)) + [(e[0], e[1]) for e in extras]:
            if x is not None:
                raise RuntimeError(f"{n} given, but the loss was built without distill=lambda")
        return None
    for n, x, k, _ in extras:
        if (x is not None) != (k > 0):
            raise RuntimeError(f"{n} given, but the loss has no such extras" if x is not None else
                               f"distill={distill}: forward needs {n} ([{k}, teacher_dim], the teacher's rows of the "
                               f"extras)")
    for n, x in list(zip(names, values)) + [(e[0], e[1]) for e in extras if e[1] is not None]:
        if x is None:
            raise RuntimeError(f"distill={distill}: forward needs {', '.join(names)}")
        if not isinstance(x, torch.Tensor) or not x.is_floating_point():
            raise RuntimeError(f"{n} must be a floating-point tensor, got "
                               f"{x.dtype if isinstance(x, torch.Tensor) else type(x).__name__}")
        if x.requires_grad:
            raise RuntimeError(f"{n} requires grad, but the teacher is frozen and no gradient flows to it: pass "
                               f"{n}.detach()")
        if x.device != image_embeddings.device:
            raise RuntimeError(f"{n} is on {x.device}, the embeddings on {image_embeddings.device}")
    timg, ttxt, tscale, tbias = values
    rows = image_embeddings.shape[0] if image_embeddings.dim() >= 1 else None
    for n, x in zip(names[:2], (timg, ttxt)):
        if x.dim() != 2 or x.shape[0] != rows or x.shape[1] < 1:
            raise RuntimeError(f"{n} must have shape [{rows}, teacher_dim], got {tuple(x.shape)}")
    if timg.shape != ttxt.shape:
        raise RuntimeError(f"{names[0]} {tuple(timg.shape)} and {names[1]} {tuple(ttxt.shape)} must have the same shape")
    for n, x in zip(names[2:], (tscale, tbias)):
        if x.numel() != 1:
            raise RuntimeError(f"{n} must be a 0-dim (1-element) tensor, got shape {tuple(x.shape)}")
    for n, x, k, side in extras:
        if x is None:
            continue
        paired = ttxt if side == "text" else timg
        if x.dim() != 2 or tuple(x.shape) != (k, timg.shape[1]):
            raise RuntimeError(f"{n} must have shape [{k}, {timg.shape[1]}] (teacher_dim), got {tuple(x.shape)}")
        if x.dtype != paired.dtype:
            raise RuntimeError(f"{n} is {x.dtype}, the paired teacher {side}s {paired.dtype}: use one dtype")
        if side == "text":
            ttxt = torch.cat([ttxt, x])
        else:
            timg = torch.cat([timg, x])
    return (_pad_dim(timg), _pad_dim(ttxt), tscale, tbias, distill)


def _teacher_extras(mod, negative_text, extra_text, extra_image):
    """The teacher-extras argument of _teacher_of for a module (DDPSigmoidLoss or SigLipLoss)."""
    return (("teacher_negative_text", negative_text, mod.hard_negatives, "text"),
            ("teacher_extra_text", extra_text, mod.extra_texts, "text"),
            ("teacher_extra_image", extra_image, mod.extra_images, "image"))


def _validate_return_metrics(return_metrics) -> None:
    if not isinstance(return_metrics, bool):
        raise RuntimeError(f"return_metrics must be a bool, got {type(return_metrics).__name__}")


def _metric_buffers(batch: int, device: torch.device, texts: Optional[int] = None, images: Optional[int] = None):
    """texts: rows of t2i_index (all T texts under extra_texts; the batch otherwise). images: rows of i2t_index (all R
    images under extra_images with ids; the batch otherwise)."""
    top1 = torch.empty(2, device=device, dtype=torch.float32)
    return (top1, torch.empty(batch if images is None else images, device=device, dtype=torch.int64),
            torch.empty(batch if texts is None else texts, device=device, dtype=torch.int64))


def _validate_return_sample_losses(return_sample_losses, distill) -> None:
    """distill: the module's distill_closed."""
    if not isinstance(return_sample_losses, bool):
        raise RuntimeError(f"return_sample_losses must be a bool, got {type(return_sample_losses).__name__}")
    if return_sample_losses and distill is not None:
        raise RuntimeError("return_sample_losses is unavailable with distill: the distillation loss kernel does not "
                           "compute per-sample losses (distill_options=True runs the one that does)")


def _sample_loss_buffers(eng) -> Tuple[torch.Tensor, torch.Tensor]:
    return (torch.empty(eng.images, device=eng.device, dtype=torch.float32),
            torch.empty(eng.texts, device=eng.device, dtype=torch.float32))


def _with_outputs(out, metric_bufs, loss_bufs):
    """(out), (out, metrics), (out, sample_losses) or (out, metrics, sample_losses), as the caller asked."""
    extra = []
    if metric_bufs is not None:
        extra.append(_metric_dict(metric_bufs))
    if loss_bufs is not None:
        extra.append({"image_loss": loss_bufs[0], "text_loss": loss_bufs[1]})
    return (out, *extra) if extra else out


def _metric_dict(bufs) -> Dict[str, torch.Tensor]:
    """The in-batch retrieval metrics of a step, as device tensors (no host synchronisation): top-1 rates of this rank's
    images / texts (0-dim fp32) and the global index of each one's best match (int64 [B]); with metrics_topk = K > 1
    also each one's K best matches (int64 [n, K]) and recall@1..K (fp32 [K]) per direction."""
    top1, i2t, t2i = bufs[:3]
    out = {"i2t_top1": top1[0], "t2i_top1": top1[1], "i2t_index": i2t, "t2i_index": t2i}
    if len(bufs) > 3:
        k, recall, i2t_topk, t2i_topk = bufs[3:]
        out.update({"i2t_topk": i2t_topk, "t2i_topk": t2i_topk, "i2t_recall": recall[:k], "t2i_recall": recall[k:]})
    return out


def _validate_metrics_topk(metrics_topk, return_metrics, distill) -> int:
    """K of a forward's top-K retrieval (None: 1, the top-1 metrics alone). distill: the module's distill_closed."""
    if metrics_topk is None:
        return 1
    if isinstance(metrics_topk, bool) or not isinstance(metrics_topk, int) or not 1 <= metrics_topk <= TOPK_MAX:
        raise RuntimeError(f"metrics_topk must be an int in 1 .. {TOPK_MAX}, got {metrics_topk!r}")
    if not return_metrics:
        raise RuntimeError("metrics_topk needs return_metrics=True")
    if distill is not None:
        raise RuntimeError("metrics_topk is unavailable with distill: the distillation loss kernel does not rank the "
                           "top K (distill_options=True runs the one that does)")
    return metrics_topk


def _topk_buffers(eng, k: int, bufs):
    """The metric buffers, followed by (K, recall [2K], i2t_topk [ni, K], t2i_topk [nt, K]) when K > 1."""
    if bufs is None or k == 1:
        return bufs
    return (*bufs, k, torch.empty(2 * k, device=eng.device, dtype=torch.float32),
            torch.empty(eng.metric_images, k, device=eng.device, dtype=torch.int64),
            torch.empty(eng.metric_texts, k, device=eng.device, dtype=torch.int64))


def _validate(image_embeddings: torch.Tensor, text_embeddings: torch.Tensor, expect_batch: Optional[int]) -> None:
    if image_embeddings.dim() != 2 or text_embeddings.dim() != 2:
        raise RuntimeError("image_embeddings and text_embeddings must be 2-D [batch, emb_dim]")
    if image_embeddings.shape != text_embeddings.shape:
        raise RuntimeError(
            f"image_embeddings {tuple(image_embeddings.shape)} and text_embeddings {tuple(text_embeddings.shape)} "
            "must have the same shape (local batch on every rank)")
    if expect_batch is not None and image_embeddings.shape[0] != expect_batch:
        # the reference fails with a broadcast RuntimeError when B != gpu_batch_size (SURVEY.md §8b)
        raise RuntimeError(
            f"The size of tensor a ({image_embeddings.shape[0]}) must match the size of tensor b ({expect_batch}): "
            "batch does not equal gpu_batch_size")
    if image_embeddings.device.type != "cuda" or text_embeddings.device != image_embeddings.device:
        raise RuntimeError("distributed_sigmoid_loss_b200 runs on CUDA (sm_90a) tensors only; there is no CPU path")


def _pad_dim(x: torch.Tensor) -> torch.Tensor:
    """Zero-pad the embedding dimension to a multiple of 8 (16-byte rows for TMA). Zero columns change no dot product;
    F.pad is differentiable, so the gradient comes back sliced to the caller's width."""
    d = x.shape[1]
    return x if d % 8 == 0 else torch.nn.functional.pad(x, (0, 8 - d % 8))


class DDPSigmoidLoss(nn.Module):
    """Drop-in for the reference ``DDPSigmoidLoss`` (distributed_sigmoid_loss.py:8-48).

    ``t_prime`` (0-dim, float64 like ``torch.tensor(np.log(10))``) and ``bias`` (0-dim fp32, -10) are
    ``nn.Parameter``s with the reference's state_dict keys; hand them to the optimizer (README.md:20).
    Embeddings are expected L2-normalised by the caller (distributed_sigmoid_loss.py:20); with
    ``normalize_inputs=False`` values must satisfy |x| <= 4094 (the gradient kernels consume fp16(16 x) copies;
    unit-norm embeddings are six orders of magnitude inside that). NaN and ±inf in the embeddings, ``t_prime`` or
    ``bias`` are never turned into finite values: the loss and each gradient element are non-finite where autograd of
    the reference is, so ``torch.amp.GradScaler`` skips the step of a tower that overflowed under autocast.
    Every rank of ``group`` must call ``forward`` the same number of times (collective, like all_gather).

    Limits (also reported by the C library when violated): all ranks of ``group`` must be GPUs of ONE node with NVLink /
    P2P access to each other (the exchange is CUDA-IPC peer memory, not NCCL), at most 32 ranks; give a multi-node job a
    per-node ``group``. A rank waiting for a peer inside a kernel gives up after ``SIGLIP_PEER_TIMEOUT_MS`` (default
    10 minutes).

    ``multi_positive=True``: every ``forward`` takes ``sample_ids`` ([B] integers, one per sample on this rank), and a pair
    is positive iff its image and text carry the same id — on any rank (repeated captions, several captions of one
    image, a sample drawn twice). Unique ids give exactly the default labels. Collective: set on every rank.

    ``forward(..., return_metrics=True)`` returns ``(loss, metrics)``: the in-batch retrieval top-1 of this rank's images
    and texts over the whole global batch (``i2t_top1``, ``t2i_top1``, 0-dim fp32) and the global index of each one's best
    match (``i2t_index``, ``t2i_index``, int64 [B]), computed by the loss kernels from the logits they already hold; a
    hit is the positional pair, or a pair with the same id under ``multi_positive``. Device tensors, no host
    synchronisation, not differentiable; loss and gradients are unchanged. Collective: every rank asks on the same steps.

    ``hard_negatives=K > 0``: every ``forward`` takes ``negative_text`` ([K, D], the dtype, device and width of the texts):
    K perturbed captions per rank that belong to no image (NegCLIP-style fine-tuning). They are scored as negatives
    against every image of the global batch, never as positives (whatever the ids), and ``negative_text.grad`` is the
    gradient of the sum over ranks of their losses. The loss still divides by the rank's image batch. ``i2t_index`` then
    ranges over all texts including the extras (global index: prefix sums of B_p + K), and a winning extra is a miss.
    Collective: every rank uses the same K.

    ``multi_positive=True, extra_texts=K > 0``: several captions per image without repeating the image. Every
    ``forward`` also takes ``extra_text`` ([K, D], like ``negative_text``) and ``extra_text_ids`` ([K] integers). Extra
    j is positive for every image of the global batch whose sample id equals ``extra_text_ids[j]``: a further caption of
    that image. An extra whose id matches no image is a hard negative. This scores ``B x (B + K)`` pairs per rank where
    repeating each image once per caption would score ``M·B x M·B``. The loss still divides by the image batch, and
    ``extra_text.grad`` comes back through autograd. With ``return_metrics``, a winning extra caption is an i2t hit,
    and ``t2i_index`` is ``[B + K]``: ``t2i_top1`` counts over every text of the rank, so a pure-negative extra is always
    a t2i miss. A caller who mixes N of them in gets the caption-only rate as ``t2i_top1 · T / (T − N)``, T = B + K.
    Cannot be combined with ``hard_negatives``. Collective: every rank uses the same K.

    ``sample_weights=True``: every ``forward`` also takes ``image_weights`` ([B]) and ``text_weights`` ([T], T = B + K
    with extras, in the order the texts are concatenated: captions, then ``negative_text`` / ``extra_text``), floating
    tensors in [0, 1] on the embeddings' device, either of them ``None`` for ones. Pair (i, j) contributes
    ``image_weights[i] · text_weights_c[j] · softplus(−y z)`` (c: the rank that owns text j), the gradients follow, and the
    loss still divides by B. A sample with both weights 0 leaves loss and gradients exactly, at the same shapes: multiply
    the loss by ``B / (B − m)`` for the mean over the m samples kept. Values outside [0, 1] are clamped into it (NaN → 0);
    larger importance weights: divide by their maximum and scale the loss by it. No gradient with respect to the weights.
    Retrieval metrics ignore the weights. Collective: set on every rank.

    ``extra_images=K > 0``: every ``forward`` also takes ``extra_image`` ([K, D], the dtype, device and width of the
    images): K more images per rank that pair with no caption position. They are scored against every text of the
    global batch and ``extra_image.grad`` comes back through autograd; the loss still divides by the paired batch B.
    Without ``multi_positive`` they are hard-negative images: every text is a negative for them. With
    ``multi_positive=True`` every forward also takes ``extra_image_ids`` ([K] integers), and extra image i is positive
    for every text of the global batch with the same id: another image of that caption (several photos of one product,
    frames of one clip, augmented crops); an id that matches no text makes it a hard-negative image. This scores
    ``(B + K) x T`` pairs per rank where repeating each caption once per image would score ``M·B x M·B``, and the images
    never leave their rank. ``image_weights`` then has B + K entries. With ``return_metrics`` a text whose best image is
    an extra is a t2i miss unless that image carries the text's id; with ids ``i2t_index`` is ``[B + K]`` and covers the
    extras (an extra whose id matches no text is always an i2t miss). Composes with ``hard_negatives`` /
    ``extra_texts``. Collective: every rank uses the same K.

    ``distill=lambda`` in (0, 1]: distillation from a frozen teacher. Every ``forward`` also takes ``teacher_image`` and
    ``teacher_text`` ([B, D_T], D_T may differ from D) and the teacher's ``teacher_t_prime`` / ``teacher_bias`` (0-dim
    device tensors, the module's own convention). The target of pair (i, j) becomes
    ``q = (1 − λ) y + λ σ(exp(t'_T) <timg_i, ttxt_j> + b_T)`` with y the hard label, and the loss
    ``(1/B) Σ w (softplus(z) − q z)``; λ = 1 is pure distillation. The teacher similarities are computed inside the loss
    kernel, tile by tile, and never stored; the teacher texts travel with the student texts. Teacher tensors follow the
    student's input rules (bf16 as is, fp32 through the fp16 conversion, ``normalize_inputs`` normalises them too) and
    must not require grad. Composes with ``multi_positive``, ``sample_weights``, ``return_metrics``, ``batch_per_rank``,
    ``sync_scalar_grads`` and both schedules. With ``distill_options=True`` it composes with every option but
    ``focal_gamma`` (the metrics and top-K lists rank the student's logits; per-sample losses sum the terms
    ``w (softplus(z) − q z)``; an excluded pair adds 0); without it, ``hard_negatives``, ``extra_texts``,
    ``extra_images``, ``exclude_groups``, ``multi_label``, ``return_sample_losses`` and ``metrics_topk`` > 1 are
    refused, as they always were. With the flag and
    ``hard_negatives`` / ``extra_texts`` / ``extra_images`` every ``forward`` also takes the teacher's rows of the extras,
    ``teacher_negative_text`` / ``teacher_extra_text`` / ``teacher_extra_image`` ([K, D_T], the same rules); a hard
    negative's target is ``λ σ(teacher logit)``, so a teacher that cannot tell it from the true caption pulls it up.
    Collective: every rank uses the same λ and D_T.

    ``forward(..., return_sample_losses=True)`` returns ``(loss, sample_losses)``, or ``(loss, metrics, sample_losses)``
    with ``return_metrics``: ``image_loss`` ([R] fp32, the paired images then the extra images) holds, for each image
    of this rank, the sum of its pair terms ``w · softplus(−y z)`` over every text of the global batch, and
    ``text_loss`` ([T] fp32, captions then ``negative_text`` / ``extra_text``) the same sum for each text over every
    image of the global batch. No 1/B is applied, so ``loss == image_loss.sum() / B`` up to rounding, and a sample of
    weight 0 reports exactly 0. The loss kernels add them up from the terms they already compute, in 64-bit fixed point,
    so they are bitwise reproducible; loss, gradients and metrics are unchanged. Device tensors, no host
    synchronisation, not differentiable; works under ``torch.no_grad()`` (data selection over a super-batch). Under
    ``distill`` they sum the distillation terms ``w (softplus(z) − q z)``. Collective: every rank asks on the same
    steps.

    ``forward(..., return_metrics=True, metrics_topk=K)``, K in 1 .. 10: with K > 1 the metrics dict also holds
    ``i2t_topk`` ([ni, K] int64: each ranked image's K best texts over the global batch, global indices, best first,
    ties to the lower index, −1 past the candidates), ``t2i_topk`` ([nt, K]: each ranked text's K best images) and
    ``i2t_recall`` / ``t2i_recall`` ([K] fp32: the fraction with a hit among the first k, k = 1 .. K, by the hit rules of
    the top-1 metrics). ``recall[0]`` and column 0 are the top-1 rate and index bit for bit; loss and gradients are
    unchanged. K = 1 or None returns today's dict. Works under ``torch.no_grad()`` (evaluation, mining). Collective: every rank asks the same K on the same steps.

    ``exclude_groups=True``: every ``forward`` also takes ``image_groups`` ([B + K_img] integers: the paired images, then
    ``extra_image``) and ``text_groups`` ([B + K] integers: the captions, then ``negative_text`` / ``extra_text``) on the
    embeddings' device; a negative group is "no group". A pair that is positive by the other options stays positive;
    any other pair whose image and text share a group (on any rank) is excluded: it adds exactly 0 to the loss, the
    gradients, ``t_prime.grad`` / ``bias.grad`` and the per-sample losses, neither pulled together nor pushed apart
    (near-duplicates, dedup clusters, class labels: in-batch false negatives). The loss still divides by B. Unique groups
    give exactly the step without the option. Retrieval metrics and top-K lists are unchanged: every pair stays a
    candidate; the lists hold global indices, so a caller can look the groups up. Works with or without
    ``multi_positive`` and with ``distill`` (an excluded pair adds 0 whatever its teacher probability). Collective: set
    on every rank.

    ``multi_label=M`` (1 <= M <= 4): multi-label positives. Every ``forward`` takes ``sample_labels`` ([B, M] integers:
    the label set of sample i, shared by image i and caption i; a negative entry is an empty slot, duplicates are
    allowed) on the embeddings' device, and with ``extra_texts=K`` / ``extra_images=K`` also ``extra_text_labels`` /
    ``extra_image_labels`` ([K, M]). ``hard_negatives`` get empty sets. A pair is positive iff it is a sample's own
    pair or its image's and text's sets share a label >= 0 (on any rank): an image labelled {golden retriever, dog} is
    a positive for the prompts "a photo of a dog" ({dog}) and "a photo of a golden retriever"; a poodle image ({poodle,
    dog}) only for the first. Every other pair is negative; the loss still divides by B. M = 1 with labels >= 0 is
    ``multi_positive`` with those ids. Retrieval metrics and top-K lists count a hit by the same rule and rank every
    image and text of the rank (extras included). Composes with every option but ``multi_positive``;
    ``exclude_groups`` applies after these positives. Collective: the same M on every rank.

    ``focal_gamma=gamma`` (0 <= gamma <= 8) and ``focal_alpha=alpha`` (None, or 0 <= alpha <= 1): torchvision's
    ``sigmoid_focal_loss`` over every pair of the global batch. With p = σ(z), target y from whatever labels the other
    options give, ``p_t = p`` if y = 1 else ``1 − p`` and ``a_t = alpha`` if y = 1 else ``1 − alpha`` (1 without
    alpha), pair (i, j) adds ``w · a_t (1 − p_t)^gamma · softplus(−(2y − 1) z)``, and the loss still divides by B: easy
    pairs, the bulk of the negatives, are down-weighted. gamma = 0 without alpha is the SigLIP loss. The terms are
    computed in the loss kernel, without the ``[B, W·B]`` logits. Excluded pairs stay 0, per-sample losses report the
    focal terms, retrieval metrics are unchanged. Derivatives below about 2⁻²⁸ lose precision in the fp16 operand of
    dimg / dtxt (DESIGN.md, "Focal pair loss"). Composes with every option but ``distill``. Collective: the same values
    on every rank.
    """

    def __init__(self, gpu_batch_size: int, group=None, cta_group: int = 2, overlap_pull: bool = True,
                 normalize_inputs: bool = False, sync_scalar_grads: bool = False, fused_step: Optional[bool] = None,
                 batch_per_rank=None, multi_positive: bool = False, hard_negatives: int = 0,
                 extra_texts: int = 0, sample_weights: bool = False, extra_images: int = 0,
                 distill: Optional[float] = None, sigma_budget_bytes: Optional[int] = None,
                 exclude_groups: bool = False, multi_label: Optional[int] = None,
                 focal_gamma: Optional[float] = None, focal_alpha: Optional[float] = None,
                 distill_options: bool = False) -> None:
        super().__init__()
        _sigma_budget_mib(sigma_budget_bytes)
        hard_negatives = _validate_hard_negatives(hard_negatives)
        extra_images = _validate_hard_negatives(extra_images, "extra_images")
        # distill_closed: what the option checks refuse, distill=lambda without distill_options (None otherwise)
        closed = None if distill_options is True else distill
        multi_label = _validate_multi_label(multi_label, multi_positive, closed)
        # extra texts carry ids under multi_positive, label sets under multi_label
        extra_texts = _validate_extra_texts(extra_texts, multi_positive or bool(multi_label), hard_negatives)
        sample_weights = _validate_sample_weights(sample_weights)
        distill = _validate_distill(distill, hard_negatives, extra_texts, extra_images, distill_options)
        self.distill_closed = None if distill_options else distill
        exclude_groups = _validate_exclude_groups(exclude_groups, self.distill_closed)
        focal = _validate_focal(focal_gamma, focal_alpha, distill)
        self.t_prime = nn.Parameter(torch.tensor(math.log(10), dtype=torch.float64))
        self.bias = nn.Parameter(torch.tensor(-10.0))
        self.gpu_batch_size = gpu_batch_size
        # extension (SURVEY.md §8f-1): take raw encoder outputs and fuse F.normalize (and its backward) around the loss
        self.normalize_inputs = normalize_inputs
        # extension (SURVEY.md §8f-2): t_prime.grad / bias.grad come back averaged over the ranks (what DDP's all-reduce
        # of the two parameters would give, README.md:20), so the module needs no DDP wrapper of its own. Collective:
        # every rank must set it, and every rank's backward must run.
        self.sync_scalar_grads = sync_scalar_grads
        # schedule: None = the fused step (two sigma operands, all flags in-kernel) when the group has more than one
        # rank, the split forward / backward otherwise (one operand either way; saves the multiply by grad_output)
        self.fused_step = fused_step
        # extension (SURVEY.md §8f-4): per-rank batch sizes may differ; every rank passes the same list
        # extension: labels from per-sample ids (positive iff same id, across ranks too)
        self.multi_positive = multi_positive
        # extension: hard-negative captions, K extra texts per rank scored against every image
        self.hard_negatives = hard_negatives
        # extension: extra captions with ids of their own (several captions per image)
        self.extra_texts = extra_texts
        # extension: per-sample loss weights (weight 0 drops a sample at a fixed batch shape)
        self.sample_weights = sample_weights
        # extension: extra images per rank (hard-negative images, or with ids several images per caption)
        self.extra_images = extra_images
        # extension: distillation from a frozen teacher (soft targets from the teacher's embeddings)
        self.distill = distill
        # extension: same-group pairs excluded from the loss (in-batch false negatives made neutral)
        self.exclude_groups = exclude_groups
        # extension: multi-label positives from per-sample label sets (0: off)
        self.multi_label = multi_label
        # extension: the focal pair loss (torchvision's sigmoid_focal_loss), (gamma, alpha) or None
        self.focal = focal
        self._cache = _EngineCache(group, cta_group, overlap_pull, sync_scalar_grads, batch_per_rank=batch_per_rank,
                                   multi_positive=multi_positive, hard_negatives=hard_negatives,
                                   extra_texts=extra_texts, sample_weights=sample_weights, extra_images=extra_images,
                                   distill=distill, sigma_budget_bytes=sigma_budget_bytes,
                                   exclude_groups=exclude_groups, multi_label=multi_label, focal=focal,
                                   distill_options=distill_options)
        # extension: bound of the 16-bit sigma operands; steps then run in row panels (memory O(budget), not O(B^2))
        self.sigma_budget_bytes = sigma_budget_bytes

    def engine_for(self, batch: int, dim: int, device: torch.device, teacher_dim: int = 0) -> SigmoidLossEngine:
        """The engine forward() uses for these shapes. A module built with distill=lambda needs the teacher's width
        (teacher_dim, padded to a multiple of 8 like dim)."""
        if (self.distill is not None) != (teacher_dim > 0):
            raise RuntimeError("engine_for: pass teacher_dim > 0 exactly when the loss was built with distill=lambda")
        return self._cache.get(batch, (dim + 7) // 8 * 8, device, (teacher_dim + 7) // 8 * 8)

    def forward(self, image_embeddings: torch.Tensor, text_embeddings: torch.Tensor, *,
                negative_text: Optional[torch.Tensor] = None, sample_ids: Optional[torch.Tensor] = None,
                return_metrics: bool = False, extra_text: Optional[torch.Tensor] = None,
                extra_text_ids: Optional[torch.Tensor] = None, image_weights: Optional[torch.Tensor] = None,
                text_weights: Optional[torch.Tensor] = None, extra_image: Optional[torch.Tensor] = None,
                extra_image_ids: Optional[torch.Tensor] = None, teacher_image: Optional[torch.Tensor] = None,
                teacher_text: Optional[torch.Tensor] = None, teacher_t_prime: Optional[torch.Tensor] = None,
                teacher_bias: Optional[torch.Tensor] = None, return_sample_losses: bool = False,
                metrics_topk: Optional[int] = None, image_groups: Optional[torch.Tensor] = None,
                text_groups: Optional[torch.Tensor] = None, sample_labels: Optional[torch.Tensor] = None,
                extra_text_labels: Optional[torch.Tensor] = None, extra_image_labels: Optional[torch.Tensor] = None,
                teacher_negative_text: Optional[torch.Tensor] = None,
                teacher_extra_text: Optional[torch.Tensor] = None,
                teacher_extra_image: Optional[torch.Tensor] = None):
        _validate_return_metrics(return_metrics)
        _validate_return_sample_losses(return_sample_losses, self.distill_closed)
        topk = _validate_metrics_topk(metrics_topk, return_metrics, self.distill_closed)
        teacher = _teacher_of(self.distill, image_embeddings,
                              ("teacher_image", "teacher_text", "teacher_t_prime", "teacher_bias"),
                              (teacher_image, teacher_text, teacher_t_prime, teacher_bias),
                              _teacher_extras(self, teacher_negative_text, teacher_extra_text, teacher_extra_image))
        ids = _validate_ids(sample_ids, self.multi_positive, image_embeddings)
        _validate_negatives(text_embeddings, negative_text, self.hard_negatives)
        _validate_negatives(text_embeddings, extra_text, self.extra_texts, "extra_text", "extra_texts")
        extra_ids = _validate_extra_text_ids(extra_text_ids, 0 if self.multi_label else self.extra_texts,
                                             text_embeddings)
        _validate_negatives(image_embeddings, extra_image, self.extra_images, "extra_image", "extra_images", "images")
        ximg_ids = _validate_extra_image_ids(extra_image_ids, self.extra_images, self.multi_positive, image_embeddings)
        weights = _weights_of(self.sample_weights, image_weights, text_weights, image_embeddings, text_embeddings,
                              self.hard_negatives + self.extra_texts, self.extra_images)
        groups = _groups_of(self.exclude_groups, image_groups, text_groups, image_embeddings, text_embeddings,
                            self.hard_negatives + self.extra_texts, self.extra_images)
        label_sets = _label_sets_of(self.multi_label, sample_labels, extra_text_labels, extra_image_labels,
                                    image_embeddings, self.extra_texts, self.extra_images)
        _validate(image_embeddings, text_embeddings, self.gpu_batch_size)
        text_embeddings = _with_negatives(_with_negatives(text_embeddings, negative_text), extra_text)
        image_embeddings = _with_negatives(image_embeddings, extra_image)
        image_embeddings, text_embeddings = _pad_dim(image_embeddings), _pad_dim(text_embeddings)
        eng = self._cache.get(self.gpu_batch_size, image_embeddings.shape[1], image_embeddings.device,
                              teacher[0].shape[1] if teacher is not None else 0)
        fused = _fused_under_budget(eng, self.fused_step)
        bufs = _metric_buffers(eng.batch, eng.device, eng.metric_texts, eng.metric_images) if return_metrics else None
        bufs = _topk_buffers(eng, topk, bufs)
        lbufs = _sample_loss_buffers(eng) if return_sample_losses else None
        loss = _SigmoidLossFn.apply(image_embeddings, text_embeddings, self.t_prime, self.bias, eng,
                                    self.normalize_inputs, fused, ids, bufs, extra_ids, weights, ximg_ids, teacher,
                                    lbufs, groups, label_sets)
        return _with_outputs(loss, bufs, lbufs)


SigmoidLoss = DDPSigmoidLoss


class SigLipLoss(nn.Module):
    """open_clip-signature adapter (rwightman_sigmoid_loss.py:12-124): scale and bias are passed in, the ring
    exchange of the original is replaced by the direct NVSwitch pulls of the fused path. ``bidir`` selects the
    visiting order of the original's bidirectional exchange (rank+1, rank-1, rank+2, ...) instead of rank+1, rank+2,
    ...; the pairs covered and the result are the same. ``multi_positive=True``: labels from the ``sample_ids`` every
    forward then takes, as in ``DDPSigmoidLoss``. ``return_metrics=True``: returns ``(loss_or_dict, metrics)`` with the
    retrieval metrics of ``DDPSigmoidLoss``; they stay out of the ``output_dict``, whose values open_clip sums into the
    total loss. ``hard_negatives=K``: every forward takes ``negative_text`` [K, D], as in ``DDPSigmoidLoss``.
    ``multi_positive=True, extra_texts=K``: every forward takes ``extra_text`` [K, D] and ``extra_text_ids`` [K], extra
    captions positive for the images with the same id, as in ``DDPSigmoidLoss`` (a pure-negative extra is always a t2i
    miss: the caption-only rate is ``t2i_top1 · T / (T − N)`` for N of them among T = B + K texts).
    ``sample_weights=True``: every forward takes ``image_weights`` [B] and ``text_weights`` [B + K] (or None for ones),
    per-sample loss weights in [0, 1] as in ``DDPSigmoidLoss``. ``extra_images=K``: every forward takes ``extra_image``
    [K, D] (and with ``multi_positive`` ``extra_image_ids`` [K]), hard-negative images or further images of a caption as
    in ``DDPSigmoidLoss``; ``image_weights`` then has B + K entries. ``distill=lambda``: every forward takes
    ``teacher_image`` / ``teacher_text`` [B, D_T] and ``teacher_logit_scale`` / ``teacher_logit_bias`` (0-dim, the
    convention of ``logit_scale`` / ``logit_bias``), distillation from a frozen teacher as in ``DDPSigmoidLoss``, with
    ``teacher_negative_text`` / ``teacher_extra_text`` / ``teacher_extra_image`` [K, D_T] for the extras.
    ``return_sample_losses=True``: also returns the per-sample losses of ``DDPSigmoidLoss`` (``image_loss`` [R],
    ``text_loss`` [T]) as the last element, after the metrics when both are asked; like the metrics they stay out of
    the ``output_dict``. ``exclude_groups=True``: every forward takes ``image_groups`` [B + K_img] and ``text_groups``
    [B + K], and same-group pairs that are not positives are excluded from the loss, as in ``DDPSigmoidLoss``.
    ``multi_label=M``: every forward takes ``sample_labels`` [B, M] (and ``extra_text_labels`` / ``extra_image_labels``
    [K, M] with ``extra_texts`` / ``extra_images``), and pairs whose label sets meet are positives, as in
    ``DDPSigmoidLoss``. ``focal_gamma`` / ``focal_alpha``: the focal pair loss of ``DDPSigmoidLoss``."""

    def __init__(self, cache_labels: bool = False, rank: int = 0, world_size: int = 1, bidir: bool = True,
                 use_horovod: bool = False, group=None, cta_group: int = 2, fused_step: Optional[bool] = None,
                 multi_positive: bool = False, hard_negatives: int = 0, extra_texts: int = 0,
                 sample_weights: bool = False, extra_images: int = 0, distill: Optional[float] = None,
                 sigma_budget_bytes: Optional[int] = None, exclude_groups: bool = False,
                 multi_label: Optional[int] = None, focal_gamma: Optional[float] = None,
                 focal_alpha: Optional[float] = None, distill_options: bool = False):
        super().__init__()
        _sigma_budget_mib(sigma_budget_bytes)
        assert not use_horovod  # same restriction as the reference (rwightman_sigmoid_loss.py:35)
        hard_negatives = _validate_hard_negatives(hard_negatives)
        extra_images = _validate_hard_negatives(extra_images, "extra_images")
        closed = None if distill_options is True else distill   # as on DDPSigmoidLoss
        multi_label = _validate_multi_label(multi_label, multi_positive, closed)
        extra_texts = _validate_extra_texts(extra_texts, multi_positive or bool(multi_label), hard_negatives)
        sample_weights = _validate_sample_weights(sample_weights)
        distill = _validate_distill(distill, hard_negatives, extra_texts, extra_images, distill_options)
        self.distill_closed = None if distill_options else distill
        exclude_groups = _validate_exclude_groups(exclude_groups, self.distill_closed)
        focal = _validate_focal(focal_gamma, focal_alpha, distill)
        self.focal = focal
        self.distill = distill
        self.exclude_groups = exclude_groups
        self.multi_label = multi_label
        self.cache_labels, self.rank, self.world_size, self.bidir = cache_labels, rank, world_size, bidir
        self.use_horovod = use_horovod
        self.fused_step = fused_step
        self.multi_positive = multi_positive
        self.hard_negatives = hard_negatives
        self.extra_texts = extra_texts
        self.sample_weights = sample_weights
        self.extra_images = extra_images
        self._cache = _EngineCache(group, cta_group, bidir=bidir, multi_positive=multi_positive,
                                   hard_negatives=hard_negatives, extra_texts=extra_texts, sample_weights=sample_weights,
                                   extra_images=extra_images, distill=distill, sigma_budget_bytes=sigma_budget_bytes,
                                   exclude_groups=exclude_groups, multi_label=multi_label, focal=focal,
                                   distill_options=distill_options)
        # bound of the 16-bit sigma operands; steps then run in row panels (as on DDPSigmoidLoss)
        self.sigma_budget_bytes = sigma_budget_bytes

    def forward(self, image_features, text_features, logit_scale, logit_bias, output_dict: bool = False, *,
                negative_text: Optional[torch.Tensor] = None, sample_ids: Optional[torch.Tensor] = None,
                return_metrics: bool = False, extra_text: Optional[torch.Tensor] = None,
                extra_text_ids: Optional[torch.Tensor] = None, image_weights: Optional[torch.Tensor] = None,
                text_weights: Optional[torch.Tensor] = None, extra_image: Optional[torch.Tensor] = None,
                extra_image_ids: Optional[torch.Tensor] = None, teacher_image: Optional[torch.Tensor] = None,
                teacher_text: Optional[torch.Tensor] = None, teacher_logit_scale: Optional[torch.Tensor] = None,
                teacher_logit_bias: Optional[torch.Tensor] = None, return_sample_losses: bool = False,
                metrics_topk: Optional[int] = None, image_groups: Optional[torch.Tensor] = None,
                text_groups: Optional[torch.Tensor] = None, sample_labels: Optional[torch.Tensor] = None,
                extra_text_labels: Optional[torch.Tensor] = None, extra_image_labels: Optional[torch.Tensor] = None,
                teacher_negative_text: Optional[torch.Tensor] = None,
                teacher_extra_text: Optional[torch.Tensor] = None,
                teacher_extra_image: Optional[torch.Tensor] = None):
        _validate_return_metrics(return_metrics)
        _validate_return_sample_losses(return_sample_losses, self.distill_closed)
        topk = _validate_metrics_topk(metrics_topk, return_metrics, self.distill_closed)
        teacher = _teacher_of(self.distill, image_features,
                              ("teacher_image", "teacher_text", "teacher_logit_scale", "teacher_logit_bias"),
                              (teacher_image, teacher_text, teacher_logit_scale, teacher_logit_bias),
                              _teacher_extras(self, teacher_negative_text, teacher_extra_text, teacher_extra_image))
        ids = _validate_ids(sample_ids, self.multi_positive, image_features)
        _validate_negatives(text_features, negative_text, self.hard_negatives)
        _validate_negatives(text_features, extra_text, self.extra_texts, "extra_text", "extra_texts")
        extra_ids = _validate_extra_text_ids(extra_text_ids, 0 if self.multi_label else self.extra_texts, text_features)
        _validate_negatives(image_features, extra_image, self.extra_images, "extra_image", "extra_images", "images")
        ximg_ids = _validate_extra_image_ids(extra_image_ids, self.extra_images, self.multi_positive, image_features)
        weights = _weights_of(self.sample_weights, image_weights, text_weights, image_features, text_features,
                              self.hard_negatives + self.extra_texts, self.extra_images)
        groups = _groups_of(self.exclude_groups, image_groups, text_groups, image_features, text_features,
                            self.hard_negatives + self.extra_texts, self.extra_images)
        label_sets = _label_sets_of(self.multi_label, sample_labels, extra_text_labels, extra_image_labels,
                                    image_features, self.extra_texts, self.extra_images)
        _validate(image_features, text_features, None)
        batch = image_features.shape[0]
        text_features = _with_negatives(_with_negatives(text_features, negative_text), extra_text)
        image_features = _with_negatives(image_features, extra_image)
        image_features, text_features = _pad_dim(image_features), _pad_dim(text_features)
        eng = self._cache.get(batch, image_features.shape[1], image_features.device,
                              teacher[0].shape[1] if teacher is not None else 0)
        if (eng.rank, eng.world) != (self.rank, self.world_size):
            raise RuntimeError(
                f"SigLipLoss(rank={self.rank}, world_size={self.world_size}) does not match the process group "
                f"(rank={eng.rank}, world_size={eng.world})")
        if logit_bias is None:
            logit_bias = torch.zeros((), device=image_features.device)
        fused = _fused_under_budget(eng, self.fused_step)
        bufs = _metric_buffers(eng.batch, eng.device, eng.metric_texts, eng.metric_images) if return_metrics else None
        bufs = _topk_buffers(eng, topk, bufs)
        lbufs = _sample_loss_buffers(eng) if return_sample_losses else None
        loss = _SigmoidLossFn.apply(image_features, text_features, logit_scale, logit_bias, eng, False, fused, ids, bufs,
                                    extra_ids, weights, ximg_ids, teacher, lbufs, groups, label_sets)
        out = {"contrastive_loss": loss} if output_dict else loss
        return _with_outputs(out, bufs, lbufs)
