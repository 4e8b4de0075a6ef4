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
                 batch_per_rank=None):
        self._L = _capi.lib()
        if not torch.cuda.is_available() or self._L.siglip_device_count() == 0:
            raise RuntimeError("distributed_sigmoid_loss_b200 needs an sm_90 (H100) device; there is no CPU fallback")
        self.batch, self.dim, self.device, self.group = batch, dim, torch.device(device), group
        self.rank, self.world = rank_world if rank_world is not None else _group_rank_world(group)
        h = ctypes.c_void_p()
        if batch_per_rank is not None:
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
        self._h = h
        _capi.check(self._L.siglip_ctx_set_option(h, _capi.SIGLIP_OPT_CTA_GROUP, int(cta_group)))
        _capi.check(self._L.siglip_ctx_set_option(h, _capi.SIGLIP_OPT_OVERLAP_PULL, int(bool(overlap_pull))))
        if self.world > 1:
            if loopback:  # single-GPU test mode: one rank of a W-rank job, peers wired to local buffers
                _capi.check(self._L.siglip_debug_loopback(h))
            else:
                self._exchange_handles()

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

    def kernel_times(self):
        """(loss_ms, loss_launches, grad_ms, grad_launches) since the last call; needs SIGLIP_OPT_KERNEL_TIMING."""
        lm, gm = ctypes.c_double(), ctypes.c_double()
        ln, gn = ctypes.c_int(), ctypes.c_int()
        _capi.check(self._L.siglip_ctx_kernel_times(self._h, ctypes.byref(lm), ctypes.byref(ln), ctypes.byref(gm),
                                                    ctypes.byref(gn)))
        return lm.value, ln.value, gm.value, gn.value

    def debug_set_text_chunk(self, chunk: int, txt: torch.Tensor) -> None:
        _capi.check(self._L.siglip_debug_set_text_chunk(self._h, chunk, txt.data_ptr(), self._stream()))

    def debug_get_slot(self, chunk: int) -> torch.Tensor:
        out = torch.empty(self.batch_per_rank[chunk], self.dim, device=self.device, dtype=torch.float32)
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
        (loss[1], dimg[B,D], dtxt[B,D], dt_prime[1], dbias[1]) for an upstream gradient of 1 (or `grad_out`, a
        1-element fp32 device tensor, multiplied in by the kernel epilogues); scalars are fp32, dimg/dtxt are
        `grad_dtype` (fp32, or bf16 written directly by the kernel epilogue)."""
        self._check(img, txt)
        self._set_grad_dtype(grad_dtype)
        opts = dict(device=self.device, dtype=torch.float32)
        scal = torch.empty(3, **opts)                 # loss, dt', dbias in one allocation
        loss, dtp, db = scal[0:1], scal[1:2], scal[2:3]
        if self._set_tprime_f64(t_prime):
            dtp = torch.empty(1, device=self.device, dtype=torch.float64)
        dimg = torch.empty(self.batch, self.dim, device=self.device, dtype=grad_dtype)
        dtxt = torch.empty(self.batch, self.dim, device=self.device, dtype=grad_dtype)
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
        dimg = torch.empty(self.batch, self.dim, device=self.device, dtype=grad_dtype)
        dtxt = torch.empty(self.batch, self.dim, device=self.device, dtype=grad_dtype)
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

    def normalize_fwd(self, x: torch.Tensor, f16: bool = False):
        """F.normalize(x, dim=1) fused with the rounding to the kernels' operand format: returns (xhat [B, D] bf16, or
        float16 holding 16*xhat with f16=True; inv_norm fp32 [B]). x: fp32 or bf16 [B, D] contiguous."""
        if tuple(x.shape) != (self.batch, self.dim) or x.dtype not in (torch.float32, torch.bfloat16) or \
                not x.is_contiguous() or x.device != self.device:
            raise RuntimeError(f"normalize_fwd expects a contiguous fp32/bf16 [{self.batch}, {self.dim}] tensor on {self.device}")
        self._set_input_f16(f16)
        xhat = torch.empty(self.batch, self.dim, device=self.device, dtype=torch.float16 if f16 else torch.bfloat16)
        inv = torch.empty(self.batch, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            _capi.check(self._L.siglip_normalize_fwd(self._h, x.data_ptr(), int(x.dtype == torch.bfloat16),
                                                     xhat.data_ptr(), inv.data_ptr(), self._stream()))
        return xhat, inv

    def normalize_bwd(self, x: torch.Tensor, inv: torch.Tensor, dxhat: torch.Tensor) -> torch.Tensor:
        """Backward of normalize_fwd: dx = inv * (dxhat - xhat <xhat, dxhat>), in x's dtype."""
        dx = torch.empty_like(x)
        with torch.cuda.device(self.device):
            _capi.check(self._L.siglip_normalize_bwd(self._h, x.data_ptr(), int(x.dtype == torch.bfloat16),
                                                     inv.data_ptr(), dxhat.data_ptr(),
                                                     int(dxhat.dtype == torch.bfloat16), dx.data_ptr(), self._stream()))
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
        """Operands are [B, D] contiguous device tensors, both bf16 (default format) or both float16 holding 16*x
        (the fp32-input format, see convert_f32); the context option follows the dtype."""
        for x in (img, txt):
            if x.device != self.device or x.dtype not in (torch.bfloat16, torch.float16) or not x.is_contiguous() or \
                    tuple(x.shape) != (self.batch, self.dim):
                raise RuntimeError(
                    f"expected contiguous bf16 (or fp16 x16) [{self.batch}, {self.dim}] tensors on {self.device}, got "
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
        if tuple(x.shape) != (self.batch, self.dim) or x.dtype != torch.float32 or not x.is_contiguous() or \
                x.device != self.device:
            raise RuntimeError(f"convert_f32 expects a contiguous fp32 [{self.batch}, {self.dim}] tensor on {self.device}")
        self._set_input_f16(f16)
        out = torch.empty(self.batch, self.dim, device=self.device, dtype=torch.float16 if f16 else torch.bfloat16)
        with torch.cuda.device(self.device):
            _capi.check(self._L.siglip_convert_f32(self._h, x.data_ptr(), out.data_ptr(), self._stream()))
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
    normalize=True additionally fuses F.normalize of both inputs (forward) and its backward around the loss."""

    @staticmethod
    def forward(ctx, img, txt, t_prime, bias, engine: SigmoidLossEngine, normalize: bool = False, fused: bool = False):
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
                # branch together, so the collective stays matched)
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
        return gi, gt, gp, gb, None, None, None


class _EngineCache:
    def __init__(self, group=None, cta_group: int = 2, overlap_pull: bool = True, sync_scalar_grads: bool = False,
                 bidir: bool = False, batch_per_rank=None):
        self.group, self.cta_group, self.overlap_pull = group, cta_group, overlap_pull
        self.sync_scalar_grads, self.bidir = sync_scalar_grads, bidir
        self.batch_per_rank = batch_per_rank
        self._engines: Dict[Tuple[int, int, int], SigmoidLossEngine] = {}

    def get(self, batch: int, dim: int, device: torch.device) -> SigmoidLossEngine:
        key = (device.index if device.index is not None else torch.cuda.current_device(), batch, dim)
        eng = self._engines.get(key)
        if eng is None:
            dev = torch.device("cuda", key[0])
            eng = SigmoidLossEngine(batch, dim, dev, self.group, self.cta_group, self.overlap_pull,
                                    batch_per_rank=self.batch_per_rank)
            if self.sync_scalar_grads:
                eng.set_option(_capi.SIGLIP_OPT_SYNC_SCALAR_GRADS, 1)
            if self.bidir:
                eng.set_option(_capi.SIGLIP_OPT_BIDIR, 1)
            self._engines[key] = eng
        return eng


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
    unit-norm embeddings are six orders of magnitude inside that).
    Every rank of ``group`` must call ``forward`` the same number of times (collective, like all_gather).

    Limits (also reported by the C library when violated): all ranks of ``group`` must be GPUs of ONE node with NVLink /
    P2P access to each other (the exchange is CUDA-IPC peer memory, not NCCL), at most 32 ranks; give a multi-node job a
    per-node ``group``. A rank waiting for a peer inside a kernel gives up after ``SIGLIP_PEER_TIMEOUT_MS`` (default
    10 minutes).
    """

    def __init__(self, gpu_batch_size: int, group=None, cta_group: int = 2, overlap_pull: bool = True,
                 normalize_inputs: bool = False, sync_scalar_grads: bool = False, fused_step: Optional[bool] = None,
                 batch_per_rank=None) -> None:
        super().__init__()
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
        self._cache = _EngineCache(group, cta_group, overlap_pull, sync_scalar_grads, batch_per_rank=batch_per_rank)

    def engine_for(self, batch: int, dim: int, device: torch.device) -> SigmoidLossEngine:
        return self._cache.get(batch, (dim + 7) // 8 * 8, device)

    def forward(self, image_embeddings: torch.Tensor, text_embeddings: torch.Tensor) -> torch.Tensor:
        _validate(image_embeddings, text_embeddings, self.gpu_batch_size)
        image_embeddings, text_embeddings = _pad_dim(image_embeddings), _pad_dim(text_embeddings)
        eng = self._cache.get(image_embeddings.shape[0], image_embeddings.shape[1], image_embeddings.device)
        fused = (eng.world > 1) if self.fused_step is None else bool(self.fused_step)
        return _SigmoidLossFn.apply(image_embeddings, text_embeddings, self.t_prime, self.bias, eng,
                                    self.normalize_inputs, fused)


SigmoidLoss = DDPSigmoidLoss


class SigLipLoss(nn.Module):
    """open_clip-signature adapter (rwightman_sigmoid_loss.py:12-124): scale and bias are passed in, the ring
    exchange of the original is replaced by the direct NVSwitch pulls of the fused path. ``bidir`` selects the
    visiting order of the original's bidirectional exchange (rank+1, rank-1, rank+2, ...) instead of rank+1, rank+2,
    ...; the pairs covered and the result are the same."""

    def __init__(self, cache_labels: bool = False, rank: int = 0, world_size: int = 1, bidir: bool = True,
                 use_horovod: bool = False, group=None, cta_group: int = 2, fused_step: Optional[bool] = None):
        super().__init__()
        assert not use_horovod  # same restriction as the reference (rwightman_sigmoid_loss.py:35)
        self.cache_labels, self.rank, self.world_size, self.bidir = cache_labels, rank, world_size, bidir
        self.use_horovod = use_horovod
        self.fused_step = fused_step
        self._cache = _EngineCache(group, cta_group, bidir=bidir)

    def forward(self, image_features, text_features, logit_scale, logit_bias, output_dict: bool = False):
        _validate(image_features, text_features, None)
        image_features, text_features = _pad_dim(image_features), _pad_dim(text_features)
        eng = self._cache.get(image_features.shape[0], image_features.shape[1], image_features.device)
        if (eng.rank, eng.world) != (self.rank, self.world_size):
            raise RuntimeError(
                f"SigLipLoss(rank={self.rank}, world_size={self.world_size}) does not match the process group "
                f"(rank={eng.rank}, world_size={eng.world})")
        if logit_bias is None:
            logit_bias = torch.zeros((), device=image_features.device)
        fused = (eng.world > 1) if self.fused_step is None else bool(self.fused_step)
        loss = _SigmoidLossFn.apply(image_features, text_features, logit_scale, logit_bias, eng, False, fused)
        return {"contrastive_loss": loss} if output_dict else loss
