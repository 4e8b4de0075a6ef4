"""ctypes binding of the C ABI declared in include/siglip_b200.h.

The shared library is built in-tree (``make -C distributed_sigmoid_loss_b200/csrc`` or
``__graft_entry__.build()``) and loaded from the package directory. There is no fallback: if the
library is missing or no sm_90 device is visible, the product path raises.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from typing import Optional

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG_DIR, "libsiglip_b200.so")
CSRC_DIR = os.path.join(_PKG_DIR, "csrc")

# every symbol include/siglip_b200.h declares (tests check the .so exports all of them)
EXPORTED_SYMBOLS = (
    "siglip_version",
    "siglip_last_error",
    "siglip_device_count",
    "siglip_ctx_create",
    "siglip_ctx_create_uneven",
    "siglip_ctx_create_texts",
    "siglip_ctx_create_extras",
    "siglip_ctx_create_distill",
    "siglip_set_teacher",
    "siglip_debug_set_teacher_text_chunk",
    "siglip_teacher_convert_f32",
    "siglip_teacher_normalize_fwd",
    "siglip_ctx_set_option",
    "siglip_ctx_workspace_bytes",
    "siglip_sigma_panel_rows",
    "siglip_ctx_sigma_panels",
    "siglip_ctx_handle_bytes",
    "siglip_ctx_export_handles",
    "siglip_ctx_import_handles",
    "siglip_forward",
    "siglip_backward",
    "siglip_ctx_saved_generation",
    "siglip_fwd_bwd",
    "siglip_fwd_bwd_scaled",
    "siglip_fwd",
    "siglip_set_sample_ids",
    "siglip_set_extra_text_ids",
    "siglip_set_extra_image_ids",
    "siglip_set_sample_weights",
    "siglip_set_groups",
    "siglip_ctx_create_labels",
    "siglip_ctx_create_distill_extras",
    "siglip_set_label_sets",
    "siglip_set_focal",
    "siglip_request_metrics",
    "siglip_request_sample_losses",
    "siglip_request_topk",
    "siglip_fwd_bwd_host",
    "siglip_convert_f32",
    "siglip_host_submit",
    "siglip_host_submit_grads",
    "siglip_host_wait",
    "siglip_scale",
    "siglip_normalize_fwd",
    "siglip_normalize_bwd",
    "siglip_normalize_fwd_rows",
    "siglip_convert_f32_rows",
    "siglip_normalize_bwd_rows",
    "siglip_ctx_kernel_times",
    "siglip_ctx_launch_count",
    "siglip_debug_gemm",
    "siglip_debug_gemm_timed",
    "siglip_debug_max_active_clusters",
    "siglip_debug_loss_max_active_clusters",
    "siglip_debug_loopback",
    "siglip_debug_set_text_chunk",
    "siglip_debug_get_slot",
    "siglip_debug_set_chunk_ids",
    "siglip_debug_set_chunk_weights",
    "siglip_debug_set_chunk_groups",
    "siglip_debug_set_chunk_label_sets",
    "siglip_debug_set_peer_extra_image_label_sets",
    "siglip_debug_set_mailbox",
    "siglip_debug_set_peer_contribution",
    "siglip_debug_set_peer_metric_keys",
    "siglip_debug_set_peer_sample_loss_partials",
    "siglip_debug_set_peer_sample_loss_poison",
    "siglip_debug_set_peer_topk_keys",
    "siglip_debug_set_peer_extra_image_ids",
    "siglip_ctx_aux_trace",
    "siglip_ctx_destroy",
)

SIGLIP_OK = 0
SIGLIP_ERR_INVALID = 1
SIGLIP_ERR_CUDA = 2
SIGLIP_ERR_NO_DEVICE = 3
SIGLIP_ERR_STATE = 4

SIGLIP_OPT_CTA_GROUP = 1
SIGLIP_OPT_OVERLAP_PULL = 2
SIGLIP_OPT_KERNEL_TIMING = 3
SIGLIP_OPT_STAGES_LOSS = 4
SIGLIP_OPT_STAGES_GRAD = 5
SIGLIP_OPT_MCAST = 6
SIGLIP_OPT_GRAD_BF16 = 7
SIGLIP_OPT_OVERLAP_REDUCE = 8
SIGLIP_OPT_EPI_SLEEP_GRAD_NS = 9
SIGLIP_OPT_EPI_SLEEP_LOSS_NS = 10
SIGLIP_OPT_SYNC_SCALAR_GRADS = 11
SIGLIP_OPT_BIDIR = 12
SIGLIP_OPT_INPUT_F16 = 13
SIGLIP_OPT_GRAD_TILE_N = 14
SIGLIP_OPT_PEER_TIMEOUT_MS = 15
SIGLIP_OPT_INKERNEL_SYNC = 16
SIGLIP_OPT_SPLIT_K = 17
SIGLIP_OPT_AUX_TRACE = 18
SIGLIP_OPT_PDL = 19
SIGLIP_OPT_TPRIME_F64 = 20
SIGLIP_OPT_SAMPLE_IDS = 21
SIGLIP_OPT_EXTRA_TEXT_IDS = 22
SIGLIP_OPT_SAMPLE_WEIGHTS = 23
SIGLIP_OPT_EXTRA_IMAGE_IDS = 24
SIGLIP_OPT_DISTILL = 25
SIGLIP_OPT_SIGMA_BUDGET_MIB = 26
SIGLIP_OPT_EXCLUDE_GROUPS = 27
SIGLIP_OPT_LABEL_SETS = 28
SIGLIP_OPT_FOCAL = 29
SIGLIP_MAX_LABELS = 4

_lib: Optional[ctypes.CDLL] = None


class SiglipError(RuntimeError):
    """A C-ABI call returned a non-zero status."""

    def __init__(self, code: int, message: str):
        super().__init__(f"siglip_b200 error {code}: {message}")
        self.code = code


def build(force: bool = False) -> str:
    """Compile the CUDA extension for sm_90a with nvcc (cross-compiles without a GPU)."""
    if force and os.path.exists(LIB_PATH):
        os.remove(LIB_PATH)
    subprocess.run(["make", "-C", CSRC_DIR], check=True, capture_output=True, text=True)
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"build did not produce {LIB_PATH}")
    return LIB_PATH


def lib() -> ctypes.CDLL:
    """Load (once) and type the shared library. Raises if it is not there."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `make -C {CSRC_DIR}` (or __graft_entry__.build()). "
            "distributed_sigmoid_loss_b200 has no CPU / PyTorch fallback."
        )
    L = ctypes.CDLL(LIB_PATH)
    vp, ci, cs = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    L.siglip_version.restype = ctypes.c_char_p
    L.siglip_last_error.restype = ctypes.c_char_p
    L.siglip_device_count.restype = ci
    L.siglip_ctx_create.argtypes = [ctypes.POINTER(vp), ci, ci, ci, ci, ci]
    L.siglip_ctx_create.restype = ci
    L.siglip_ctx_set_option.argtypes = [vp, ci, ci]
    L.siglip_ctx_set_option.restype = ci
    L.siglip_ctx_workspace_bytes.argtypes = [vp]
    L.siglip_ctx_workspace_bytes.restype = cs
    L.siglip_sigma_panel_rows.argtypes = [ci, ci, ci, ci, ci, ci, ctypes.POINTER(ci)]
    L.siglip_sigma_panel_rows.restype = ci
    L.siglip_ctx_sigma_panels.argtypes = [vp, ci, ctypes.POINTER(ci), ctypes.POINTER(ci), ctypes.POINTER(ci)]
    L.siglip_ctx_sigma_panels.restype = ci
    L.siglip_ctx_handle_bytes.restype = cs
    L.siglip_ctx_export_handles.argtypes = [vp, vp, cs]
    L.siglip_ctx_export_handles.restype = ci
    L.siglip_ctx_import_handles.argtypes = [vp, vp, cs]
    L.siglip_ctx_import_handles.restype = ci
    L.siglip_forward.argtypes = [vp, vp, vp, vp, vp, vp, ci, vp]
    L.siglip_forward.restype = ci
    L.siglip_backward.argtypes = [vp] * 10
    L.siglip_backward.restype = ci
    L.siglip_ctx_saved_generation.argtypes = [vp]
    L.siglip_ctx_saved_generation.restype = ctypes.c_ulonglong
    L.siglip_fwd_bwd.argtypes = [vp] * 11
    L.siglip_fwd_bwd.restype = ci
    L.siglip_fwd_bwd_scaled.argtypes = [vp] * 12
    L.siglip_fwd_bwd_scaled.restype = ci
    L.siglip_ctx_create_uneven.argtypes = [ctypes.POINTER(vp), ci, ci, ci, ctypes.POINTER(ci), ci]
    L.siglip_ctx_create_uneven.restype = ci
    L.siglip_ctx_create_texts.argtypes = [ctypes.POINTER(vp), ci, ci, ci, ctypes.POINTER(ci), ctypes.POINTER(ci), ci]
    L.siglip_ctx_create_texts.restype = ci
    L.siglip_ctx_create_extras.argtypes = [ctypes.POINTER(vp), ci, ci, ci, ctypes.POINTER(ci), ctypes.POINTER(ci),
                                           ctypes.POINTER(ci), ci]
    L.siglip_ctx_create_extras.restype = ci
    L.siglip_ctx_create_distill.argtypes = [ctypes.POINTER(vp), ci, ci, ci, ctypes.POINTER(ci), ci, ci]
    L.siglip_ctx_create_distill.restype = ci
    L.siglip_set_teacher.argtypes = [vp, vp, vp, ci, vp, vp, ctypes.c_float]
    L.siglip_set_teacher.restype = ci
    L.siglip_debug_set_teacher_text_chunk.argtypes = [vp, ci, vp, vp]
    L.siglip_debug_set_teacher_text_chunk.restype = ci
    L.siglip_teacher_convert_f32.argtypes = [vp, ci, vp, vp, ci, vp]
    L.siglip_teacher_convert_f32.restype = ci
    L.siglip_teacher_normalize_fwd.argtypes = [vp, ci, vp, ci, vp, vp, ci, vp]
    L.siglip_teacher_normalize_fwd.restype = ci
    L.siglip_set_extra_image_ids.argtypes = [vp, vp, vp]
    L.siglip_set_extra_image_ids.restype = ci
    L.siglip_debug_set_peer_extra_image_ids.argtypes = [vp, ci, vp, vp]
    L.siglip_debug_set_peer_extra_image_ids.restype = ci
    L.siglip_host_submit_grads.argtypes = [vp, vp, vp, ctypes.c_float, ctypes.c_float, vp, vp,
                                           ctypes.POINTER(ctypes.c_ulonglong), vp]
    L.siglip_host_submit_grads.restype = ci
    L.siglip_debug_set_mailbox.argtypes = [vp, ci, ctypes.c_float, ctypes.c_float]
    L.siglip_debug_set_mailbox.restype = ci
    L.siglip_debug_set_peer_contribution.argtypes = [vp, ci, vp, vp]
    L.siglip_debug_set_peer_contribution.restype = ci
    L.siglip_ctx_aux_trace.argtypes = [vp, vp, ci, ctypes.POINTER(ci)]
    L.siglip_ctx_aux_trace.restype = ci
    L.siglip_fwd.argtypes = [vp] * 7
    L.siglip_fwd.restype = ci
    L.siglip_fwd_bwd_host.argtypes = [vp, vp, vp, ctypes.c_float, ctypes.c_float, vp, vp, vp, vp, vp, vp]
    L.siglip_fwd_bwd_host.restype = ci
    L.siglip_convert_f32.argtypes = [vp, vp, vp, vp]
    L.siglip_convert_f32.restype = ci
    L.siglip_host_submit.argtypes = [vp, vp, vp, ctypes.c_float, ctypes.c_float,
                                     ctypes.POINTER(ctypes.c_ulonglong), vp]
    L.siglip_host_submit.restype = ci
    L.siglip_host_wait.argtypes = [vp, ctypes.c_ulonglong, vp, vp, vp]
    L.siglip_host_wait.restype = ci
    L.siglip_normalize_fwd.argtypes = [vp, vp, ci, vp, vp, vp]
    L.siglip_normalize_fwd.restype = ci
    L.siglip_normalize_bwd.argtypes = [vp, vp, ci, vp, vp, ci, vp, vp]
    L.siglip_normalize_bwd.restype = ci
    L.siglip_normalize_fwd_rows.argtypes = [vp, ci, vp, ci, vp, vp, vp]
    L.siglip_normalize_fwd_rows.restype = ci
    L.siglip_convert_f32_rows.argtypes = [vp, ci, vp, vp, vp]
    L.siglip_convert_f32_rows.restype = ci
    L.siglip_normalize_bwd_rows.argtypes = [vp, ci, vp, ci, vp, vp, ci, vp, vp]
    L.siglip_normalize_bwd_rows.restype = ci
    L.siglip_scale.argtypes = [vp, vp, vp, cs, ci, vp, vp]
    L.siglip_scale.restype = ci
    L.siglip_ctx_kernel_times.argtypes = [vp, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ci),
                                          ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ci)]
    L.siglip_ctx_kernel_times.restype = ci
    L.siglip_debug_loopback.argtypes = [vp]
    L.siglip_debug_loopback.restype = ci
    L.siglip_debug_set_text_chunk.argtypes = [vp, ci, vp, vp]
    L.siglip_debug_set_text_chunk.restype = ci
    L.siglip_debug_get_slot.argtypes = [vp, ci, vp, vp]
    L.siglip_debug_get_slot.restype = ci
    L.siglip_set_sample_ids.argtypes = [vp, vp, vp]
    L.siglip_set_sample_ids.restype = ci
    L.siglip_set_extra_text_ids.argtypes = [vp, vp, vp]
    L.siglip_set_extra_text_ids.restype = ci
    L.siglip_debug_set_chunk_ids.argtypes = [vp, ci, vp, vp]
    L.siglip_debug_set_chunk_ids.restype = ci
    L.siglip_set_sample_weights.argtypes = [vp, vp, vp, vp]
    L.siglip_set_sample_weights.restype = ci
    L.siglip_debug_set_chunk_weights.argtypes = [vp, ci, vp, vp]
    L.siglip_debug_set_chunk_weights.restype = ci
    L.siglip_set_groups.argtypes = [vp, vp, vp, vp]
    L.siglip_set_groups.restype = ci
    L.siglip_debug_set_chunk_groups.argtypes = [vp, ci, vp, vp]
    L.siglip_debug_set_chunk_groups.restype = ci
    L.siglip_ctx_create_labels.argtypes = [ctypes.POINTER(vp), ci, ci, ci, ctypes.POINTER(ci), ctypes.POINTER(ci),
                                           ctypes.POINTER(ci), ci, ci]
    L.siglip_ctx_create_labels.restype = ci
    L.siglip_ctx_create_distill_extras.argtypes = [ctypes.POINTER(vp), ci, ci, ci, ctypes.POINTER(ci),
                                                   ctypes.POINTER(ci), ctypes.POINTER(ci), ci, ci, ci]
    L.siglip_ctx_create_distill_extras.restype = ci
    L.siglip_set_label_sets.argtypes = [vp, vp, vp, vp, vp]
    L.siglip_set_label_sets.restype = ci
    L.siglip_set_focal.argtypes = [vp, ctypes.c_float, ctypes.c_float]
    L.siglip_set_focal.restype = ci
    L.siglip_debug_set_chunk_label_sets.argtypes = [vp, ci, vp, vp]
    L.siglip_debug_set_chunk_label_sets.restype = ci
    L.siglip_debug_set_peer_extra_image_label_sets.argtypes = [vp, ci, vp, vp]
    L.siglip_debug_set_peer_extra_image_label_sets.restype = ci
    L.siglip_request_metrics.argtypes = [vp, vp, vp, vp]
    L.siglip_request_metrics.restype = ci
    L.siglip_debug_set_peer_metric_keys.argtypes = [vp, ci, vp, vp]
    L.siglip_debug_set_peer_metric_keys.restype = ci
    L.siglip_request_sample_losses.argtypes = [vp, vp, vp]
    L.siglip_request_sample_losses.restype = ci
    L.siglip_debug_set_peer_sample_loss_partials.argtypes = [vp, ci, vp, vp]
    L.siglip_debug_set_peer_sample_loss_partials.restype = ci
    L.siglip_debug_set_peer_sample_loss_poison.argtypes = [vp, ci, vp, vp]
    L.siglip_debug_set_peer_sample_loss_poison.restype = ci
    L.siglip_request_topk.argtypes = [vp, ci, vp, vp, vp]
    L.siglip_request_topk.restype = ci
    L.siglip_debug_set_peer_topk_keys.argtypes = [vp, ci, vp, vp]
    L.siglip_debug_set_peer_topk_keys.restype = ci
    L.siglip_ctx_launch_count.argtypes = [vp]
    L.siglip_ctx_launch_count.restype = ctypes.c_ulonglong
    L.siglip_debug_gemm.argtypes = [ci, ci, ci, ci, ci, vp, ctypes.c_longlong, ci, vp, ctypes.c_longlong, ci, vp,
                                    ctypes.c_longlong, vp]
    L.siglip_debug_gemm.restype = ci
    L.siglip_debug_gemm_timed.argtypes = [ci, ci, ci, ci, ci, vp, ctypes.c_longlong, ci, vp, ctypes.c_longlong, ci, vp,
                                          ctypes.c_longlong, ci, ctypes.POINTER(ctypes.c_float), vp]
    L.siglip_debug_gemm_timed.restype = ci
    L.siglip_debug_max_active_clusters.argtypes = [ci, ci, ci, ci, ci]
    L.siglip_debug_max_active_clusters.restype = ci
    L.siglip_debug_loss_max_active_clusters.argtypes = [ci, ci, ci, ci, ci]
    L.siglip_debug_loss_max_active_clusters.restype = ci
    L.siglip_ctx_destroy.argtypes = [vp]
    L.siglip_ctx_destroy.restype = None
    _lib = L
    return L


def last_error() -> str:
    return lib().siglip_last_error().decode("utf-8", "replace")


def check(code: int) -> None:
    if code != SIGLIP_OK:
        raise SiglipError(code, last_error())


def max_active_clusters(cta_group: int, mcast: int, tile_n: int, stages: int = 0, device: int = 0) -> int:
    """Clusters of the persistent grid of a gradient-kernel launch on `device` (siglip_debug_max_active_clusters)."""
    n = lib().siglip_debug_max_active_clusters(device, cta_group, mcast, tile_n, stages)
    if n < 0:
        raise SiglipError(-n, last_error())
    return n


# the loss kernel's modes by number (csrc/siglip_kernels.cuh KernelMode)
LOSS_MODES = {"loss": 0, "distill": 2, "sample_loss": 3, "topk": 4, "groups": 5, "labels": 6, "focal": 7,
              "distill_opts": 8}


def loss_max_active_clusters(mode: str, cta_group: int, mcast: int, stages: int = 0, device: int = 0) -> int:
    """Clusters of the persistent grid of a loss-kernel launch of `mode` (a LOSS_MODES name) on `device`
    (siglip_debug_loss_max_active_clusters)."""
    n = lib().siglip_debug_loss_max_active_clusters(device, cta_group, mcast, LOSS_MODES[mode], stages)
    if n < 0:
        raise SiglipError(-n, last_error())
    return n


def device_count() -> int:
    return int(lib().siglip_device_count())


def version() -> str:
    return lib().siglip_version().decode()
