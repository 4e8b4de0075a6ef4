"""H100-native distributed sigmoid (SigLIP) loss: drop-in for ahmdtaha/distributed_sigmoid_loss's
``DDPSigmoidLoss`` hot path, computed by hand-written sm_90a kernels behind a C ABI
(include/siglip_b200.h). Importing the package does not need a GPU; running the loss does."""
from . import _capi
from .loss import DDPSigmoidLoss, SigLipLoss, SigmoidLoss, SigmoidLossEngine, chunk_schedule

__all__ = ["DDPSigmoidLoss", "SigmoidLoss", "SigLipLoss", "SigmoidLossEngine", "chunk_schedule", "_capi"]
__version__ = "0.4.0"
