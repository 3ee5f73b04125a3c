"""hcp_diffusion_b200 -- H100-native (sm_90a) UNet denoising hot path behind HCP-Diffusion's plugin surface.

Only the hot path of the reference (IrisRainbowNeko/HCP-Diffusion) is provided: the SD1.x `UNet2DConditionModel`
forward/backward with layer-wise LoRA adapters, the cfg-driven layer selection (`make_hcpdiff`, `re:` patterns), the LoRA
checkpoint format, and the data-parallel training step.  All arithmetic runs in the hand-written CUDA library
`lib/libhcpb200.so` (C ABI: include/hcp_b200.h); there is no CPU or eager fallback.
"""
from . import _lib  # noqa: F401
from ._lib import HcpError, build  # noqa: F401

__version__ = "0.1.0"
