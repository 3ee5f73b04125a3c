"""Layer-wise LoRA adapters with hcpdiff's plugin surface, executed by the fused sm_90a kernels.

Same classes, constructor signatures, parameter names and checkpoint keys as the reference's active implementation
(hcpdiff/models/lora_base_patch.py: LoraPatchContainer :20-35, LoraBlock :37-156, LoraGroup :175-194;
hcpdiff/models/lora_layers_patch.py: LoraLayer :21, LinearLayer :25-62, lora_layer_map :218-221):

    <layer>._host.weight                        frozen base weight (the container stores the host as `_host`)
    <layer>.lora_block_<id>.layer.W_down [r,in] trainable
    <layer>.lora_block_<id>.layer.W_up  [out,r] trainable
    <layer>.lora_block_<id>.alpha       []      buffer = alpha / rank (alpha_auto_scale) or alpha

Semantics: y = x @ (W_host + sum_b alpha_b * W_up_b @ W_down_b)^T + bias.  The reference materialises the [out,in] delta
every forward (lora_base_patch.py:61-62, lora_layers_patch.py:44-45); here the delta stays factored and rides the same
tensor-core pipeline as extra K-blocks (csrc/gemm.cu).

Also here: `Conv2dLayer` (LoCon, lora_layers_patch.py:64-100: W_down [r,in,kh,kw], W_up [out,r,1,1]) and the DreamArtist++
pair `DAPPLayer` / `DAPPPatchContainer` (lora_layers_patch.py:102-216: 'n' blocks act on the first half of the batch, 'p' blocks
on the second).  Supported on this path: nn.Linear and Conv2d hosts, dropout == 0, no LoRA bias.
"""
from __future__ import annotations

import math
from typing import Dict, Union

import torch
from torch import nn

from .plugin import PatchPluginBlock, PatchPluginContainer, PluginGroup


class LoraPatchContainer(PatchPluginContainer):
    def forward(self, x, *args, **kwargs):
        """Stand-alone call of one patched layer (inside the UNet the parent block fuses several layers into one GEMM and
        does not come through here).  Extra positional arguments (diffusers' `scale`) are ignored like in the reference."""
        from ..runtime import ConvGroup, LinearGroup  # local import: runtime imports this module
        grp = self.__dict__.get("_hcp_group")
        if grp is None:
            host = self._host
            is3x3 = isinstance(host, nn.Conv2d) and host.kernel_size == (3, 3)
            grp = ConvGroup(self) if is3x3 else LinearGroup([self])
            self.__dict__["_hcp_group"] = grp
        return grp.run_standalone(x)


class LoraBlock(PatchPluginBlock):
    container_cls = LoraPatchContainer
    wrapable_classes = (nn.Linear, nn.Conv2d)

    def __init__(self, lora_id: int, host: Union[nn.Linear, nn.Conv2d], rank, dropout=0.1, alpha=1.0, bias=False,
                 alpha_auto_scale=True, parent_block=None, host_name=None, **kwargs):
        super().__init__(f"lora_block_{lora_id}", host, parent_block=parent_block, host_name=host_name)
        self.bias = bias
        host = self.host()
        if isinstance(host, nn.Linear):
            self.host_type = "linear"
            self.layer = self.LinearLayer(host, rank, bias, self)
        elif isinstance(host, nn.Conv2d):
            self.host_type = "conv"
            self.layer = self.Conv2dLayer(host, rank, bias, self)
        else:
            raise NotImplementedError(f"No lora for {type(host)}")
        if bias:
            raise NotImplementedError("LoRA bias is not supported on the H100 hot path")
        self.dropout = nn.Dropout(dropout)
        self.rank = self.layer.rank
        self.register_buffer("alpha", torch.tensor(alpha / self.rank if alpha_auto_scale else alpha))

    def get_weight(self):
        return self.layer.get_weight() * self.alpha

    def get_bias(self):
        return None

    def init_weights(self, svd_init=False):
        if svd_init:
            raise NotImplementedError("svd_init is broken in the reference's patch variant (SURVEY.md App. C.3) and is not provided")
        self.layer.reset_parameters()

    class LinearLayer(nn.Module):
        def __init__(self, host: nn.Linear, rank, bias, block):
            super().__init__()
            self.rank = rank
            if isinstance(self.rank, float):
                self.rank = max(round(host.out_features * self.rank), 1)

    class Conv2dLayer(nn.Module):
        def __init__(self, host: nn.Conv2d, rank, bias, block):
            super().__init__()
            self.rank = rank
            if isinstance(self.rank, float):
                self.rank = max(round(host.out_channels * self.rank), 1)

    @classmethod
    def wrap_layer(cls, lora_id: int, layer, rank=1, dropout=0.0, alpha=1.0, svd_init=False, bias=False, mask=None, **kwargs):
        block = cls(lora_id, layer, rank, dropout, alpha, bias=bias, **kwargs)
        block.init_weights(svd_init)
        return block

    @classmethod
    def wrap_model(cls, lora_id: int, model: nn.Module, **kwargs):
        return super(LoraBlock, cls).wrap_model(lora_id, model, exclude_classes=(LoraBlock,), **kwargs)

    # ---- state helpers used by the checkpoint managers (reference lora_base_patch.py:158-173) -------------------------
    @staticmethod
    def extract_lora_state(model: nn.Module):
        return {k: v for k, v in model.state_dict().items() if "lora_block_" in k}

    @staticmethod
    def extract_state_without_lora(model: nn.Module):
        return {k: v for k, v in model.state_dict().items() if "lora_block_" not in k}

    @staticmethod
    def extract_param_without_lora(model: nn.Module):
        return {k: v for k, v in model.named_parameters() if "lora_block_" not in k}

    @staticmethod
    def extract_trainable_state_without_lora(model: nn.Module):
        trainable = {k for k, v in model.named_parameters() if v.requires_grad}
        return {k: v for k, v in model.state_dict().items() if k in trainable and "lora_block_" not in k}


class LoraLayer(LoraBlock):
    def __init__(self, lora_id: int, host, rank=1, dropout=0.1, alpha=1.0, bias=False, alpha_auto_scale=True, **kwargs):
        super().__init__(lora_id, host, rank, dropout, alpha=alpha, bias=bias, alpha_auto_scale=alpha_auto_scale, **kwargs)

    class LinearLayer(LoraBlock.LinearLayer):
        def __init__(self, host: nn.Linear, rank, bias, block):
            super().__init__(host, rank, bias, block)
            dev = host.weight.device
            self.W_down = nn.Parameter(torch.empty(self.rank, host.in_features, device=dev))
            self.W_up = nn.Parameter(torch.empty(host.out_features, self.rank, device=dev))
            self.register_parameter("bias", None)

        def reset_parameters(self):
            nn.init.kaiming_uniform_(self.W_down, a=math.sqrt(5))
            nn.init.zeros_(self.W_up)

        def get_weight(self) -> torch.Tensor:
            return torch.mm(self.W_up, self.W_down)

        def get_collapsed_param(self):
            return self.W_up.data @ self.W_down.data, None


    class Conv2dLayer(LoraBlock.Conv2dLayer):
        def __init__(self, host: nn.Conv2d, rank, bias, block):
            super().__init__(host, rank, bias, block)
            if host.groups != 1 or host.dilation != (1, 1):
                raise NotImplementedError("Conv2d LoRA on grouped / dilated convolutions is not supported on the H100 hot path")
            dev = host.weight.device
            self.W_down = nn.Parameter(torch.empty(self.rank, host.in_channels, *host.kernel_size, device=dev))
            self.W_up = nn.Parameter(torch.empty(host.out_channels, self.rank, 1, 1, device=dev))
            self.register_parameter("bias", None)
            self.stride, self.padding, self.dilation, self.groups = host.stride, host.padding, host.dilation, host.groups

        def reset_parameters(self):
            nn.init.kaiming_uniform_(self.W_down, a=math.sqrt(5))
            nn.init.zeros_(self.W_up)

        def get_weight(self) -> torch.Tensor:
            return torch.einsum("or...,ri...->oi...", self.W_up[:, :, 0, 0], self.W_down)

        def get_collapsed_param(self):
            return torch.einsum("or,rikl->oikl", self.W_up.data[:, :, 0, 0], self.W_down.data), None


class DAPPPatchContainer(LoraPatchContainer):
    """DreamArtist++ container (reference lora_layers_patch.py:102-133): the input batch is [negative half | positive half];
    rows of the first half get W_host + sum of the branch-'n' deltas, rows of the second half the branch-'p' deltas."""


class DAPPLayer(LoraLayer):
    """LoRA block bound to one CFG branch (reference lora_layers_patch.py:135-216).  Same parameters / checkpoint keys as
    LoraLayer; `branch` is 'p' (positive prompt half) or 'n' (negative half)."""
    container_cls = DAPPPatchContainer

    def __init__(self, lora_id: int, host, rank=1, dropout=0.1, alpha=1.0, bias=False, alpha_auto_scale=True, branch="p", **kwargs):
        if branch not in ("p", "n"):
            raise ValueError(f"DAPPLayer branch must be 'p' or 'n', got {branch!r}")
        super().__init__(lora_id, host, rank, dropout, alpha=alpha, bias=bias, alpha_auto_scale=alpha_auto_scale, **kwargs)
        self.branch = branch


class LoraGroup(PluginGroup):
    def set_inplace(self, inplace):
        for item in self.plugin_dict.values():
            item.set_hyper_params(inplace=inplace)


lora_layer_map: Dict[str, type] = {
    "lora": LoraLayer,
    "dapp": DAPPLayer,
}
