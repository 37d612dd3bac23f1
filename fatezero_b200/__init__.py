"""fatezero_b200 — H100-native (sm_90a) implementation of FateZero's DDIM-inversion + attention-fused denoising hot path.

    from fatezero_b200 import UNetPseudo3DConditionModel, P2pDDIMSpatioTemporalPipeline, DDIMScheduler
    (or the reference's own import paths through the `video_diffusion` alias package)

Compute runs in libfatezero_b200.so (hand-written CUDA, C ABI in include/fatezero_b200.h); there is no CPU fallback."""
from .controllers import (AttentionControlEdit, AttentionRefine, AttentionReplace, AttentionReweight, AttentionStore,  # noqa: F401
                          EmptyControl, make_controller, register_attention_control)
from .pipeline import P2pDDIMSpatioTemporalPipeline  # noqa: F401
from .scheduler import DDIMScheduler  # noqa: F401
from .spatial_blend import SpatialBlender  # noqa: F401
from .unet import UNetPseudo3DConditionModel  # noqa: F401

__version__ = "0.1.0"
