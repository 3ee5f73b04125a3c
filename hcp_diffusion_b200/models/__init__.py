from .plugin import BasePluginBlock, PatchPluginBlock, PatchPluginContainer, PluginGroup, WrapablePlugin  # noqa: F401
from .lora import LoraBlock, LoraGroup, LoraLayer, LoraPatchContainer, lora_layer_map  # noqa: F401
from .unet import UNet2DConditionModel  # noqa: F401
from .clip import CLIPTextModel, CLIPTextModelWithProjection, SDXLTextEncoder, encode_prompt, encode_prompt_sdxl  # noqa: F401
