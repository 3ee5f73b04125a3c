from .plugin import BasePluginBlock, PatchPluginBlock, PatchPluginContainer, PluginGroup, WrapablePlugin  # noqa: F401
from .lora import LoraBlock, LoraGroup, LoraLayer, LoraPatchContainer, lora_layer_map  # noqa: F401
from .unet import UNet2DConditionModel  # noqa: F401
from .clip import CLIPTextModel, encode_prompt  # noqa: F401
