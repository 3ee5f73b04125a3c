"""AdamW8bit over the flat parameter buffer: option parsing, the two code maps and the device tables of `hcp_adamw8bit_flat`.

The optimizer is `bitsandbytes.optim.AdamW8bit` (Optimizer2State with optim_bits 8, block_wise True).  A tensor with at least
`min_8bit_size` elements keeps both Adam moments as 8-bit codes, one code per element, plus one fp32 scale (absmax) per 256-element
block counted from the tensor's own first element; the first moment decodes through the signed dynamic map, the second through the
unsigned one.  A smaller tensor keeps fp32 moments.  The kernel (csrc/optim.cu) walks the tensors in items of whole blocks; this
module cuts them and lays out the state buffers:

  codes    uint8 [2, code_bytes]: the first moment's codes, then the second's; a tensor's codes start at a multiple of 16
  absmax   fp32 [2, nblocks]: the block scales of the first moment, then the second's
  state32  fp32 [2, small_numel]: m, then v, of the tensors below min_8bit_size; each starts at a multiple of 4
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np
import torch

# bitsandbytes.optim.AdamW8bit.__init__ keywords and defaults (optim_bits is forced to 8 by the class)
DEFAULTS = {"lr": 1e-3, "betas": (0.9, 0.999), "eps": 1e-8, "weight_decay": 1e-2, "amsgrad": False, "optim_bits": 32, "args": None,
            "min_8bit_size": 4096, "percentile_clipping": 100, "block_wise": True, "is_paged": False}
BLOCK = 256             # elements per absmax block (and per work block of a 32-bit tensor)
ITEM_BLOCKS = 64        # blocks per work item: one CTA walks an item four blocks at a time
MODE_32BIT, MODE_8BIT = 0, 1

TENSOR_DTYPE = np.dtype([("offset", "<i8"), ("numel", "<i8"), ("state", "<i8"), ("absmax", "<i8"), ("mode", "<i4"), ("group", "<i4")])
ITEM_DTYPE = np.dtype([("tensor", "<i4"), ("block0", "<i4"), ("block1", "<i4"), ("pad", "<i4")])


def check_options(kw: Optional[dict]) -> dict:
    """The constructor keys of bitsandbytes' AdamW8bit with its defaults.  An unknown key is a TypeError (as the constructor raises);
    the options this engine does not implement are refused with NotImplementedError."""
    kw = dict(kw or {})
    unknown = sorted(set(kw) - set(DEFAULTS))
    if unknown:
        raise TypeError(f"AdamW8bit.__init__() got unexpected keyword arguments {unknown}")
    out = {**DEFAULTS, **kw}
    refused = [("percentile_clipping", out["percentile_clipping"] != 100), ("block_wise", not out["block_wise"]),
               ("amsgrad", bool(out["amsgrad"])), ("is_paged", bool(out["is_paged"])), ("args", out["args"] is not None)]
    for key, bad in refused:
        if bad:
            raise NotImplementedError(f"bitsandbytes.optim.AdamW8bit with {key}={out[key]!r} is not supported (percentile clipping, "
                                      "non-blockwise and paged state, AMSGrad and an args override are not implemented)")
    betas = tuple(float(b) for b in out["betas"])
    if len(betas) != 2:
        raise ValueError(f"AdamW8bit betas {out['betas']!r}: two values (beta1, beta2)")
    if int(out["min_8bit_size"]) < 0:
        raise ValueError(f"min_8bit_size {out['min_8bit_size']!r} must be >= 0")
    return {"lr": float(out["lr"]), "betas": betas, "eps": float(out["eps"]), "weight_decay": float(out["weight_decay"]),
            "min_8bit_size": int(out["min_8bit_size"])}


def create_dynamic_map(signed: bool = True, max_exponent_bits: int = 7, total_bits: int = 8) -> torch.Tensor:
    """bitsandbytes.functional.create_dynamic_map: 256 sorted fp32 values in [-1, 1] (signed) or [0, 1] (unsigned).  Per decade
    10^(i-6), i = 0..6, the midpoints of torch.linspace(0.1, 1, 2^i + 1) (signed, with their negatives) or of 2^(i+1) + 1 points
    (unsigned), then 0 and 1.  Computed in torch's fp32 exactly as there, so the values match the library's bit for bit."""
    data = []
    non_sign_bits = total_bits - 1
    additional_items = 2 ** (non_sign_bits - max_exponent_bits) - 1
    for i in range(max_exponent_bits):
        fraction_items = int(2 ** (i + non_sign_bits - max_exponent_bits) + 1 if signed
                             else 2 ** (i + non_sign_bits - max_exponent_bits + 1) + 1)
        boundaries = torch.linspace(0.1, 1, fraction_items, dtype=torch.float32)
        means = (boundaries[:-1] + boundaries[1:]) / 2.0
        data += ((10 ** (-(max_exponent_bits - 1) + i)) * means).tolist()
        if signed:
            data += (-(10 ** (-(max_exponent_bits - 1) + i)) * means).tolist()
    if additional_items > 0:
        boundaries = torch.linspace(0.1, 1, additional_items + 1, dtype=torch.float32)
        means = (boundaries[:-1] + boundaries[1:]) / 2.0
        data += ((10 ** (-(max_exponent_bits - 1) + max_exponent_bits - 1)) * means).tolist()
        if signed:
            data += (-(10 ** (-(max_exponent_bits - 1) + max_exponent_bits - 1)) * means).tolist()
    data.append(0)
    data.append(1.0)
    assert len(data) == 2 ** total_bits
    data += [0] * (256 - len(data))
    data.sort()
    return torch.tensor(data, dtype=torch.float32)


def maps() -> torch.Tensor:
    """fp32 [2, 256]: the signed map (first moment), then the unsigned one (second moment)."""
    return torch.stack([create_dynamic_map(True), create_dynamic_map(False)])


class Layout:
    """Tensor table, work items and state sizes for tensors of `numels` at flat `offsets`, tensor i in parameter group `groups[i]`;
    a tensor with at least `min_8bit_size` elements is 8-bit."""

    def __init__(self, numels: Sequence[int], offsets: Sequence[int], groups: Sequence[int], min_8bit_size: int = 4096):
        tens = np.zeros(len(numels), dtype=TENSOR_DTYPE)
        items = []
        code, blocks, small = 0, 0, 0
        for i, (n, off, grp) in enumerate(zip(numels, offsets, groups)):
            n = int(n)
            if n <= 0:
                raise ValueError(f"tensor {i}: empty")
            t = tens[i]
            nb = -(-n // BLOCK)
            t["offset"], t["numel"], t["group"] = off, n, grp
            if n >= min_8bit_size:
                t["mode"], t["state"], t["absmax"] = MODE_8BIT, code, blocks
                code += -(-n // 16) * 16
                blocks += nb
            else:
                t["mode"], t["state"], t["absmax"] = MODE_32BIT, small, -1
                small += -(-n // 4) * 4
            b0 = np.arange(0, nb, ITEM_BLOCKS)
            it = np.zeros(b0.size, dtype=ITEM_DTYPE)
            it["tensor"], it["block0"], it["block1"] = i, b0, np.minimum(b0 + ITEM_BLOCKS, nb)
            items.append(it)
        self.tensors = tens
        self.items = np.concatenate(items) if items else np.zeros(0, dtype=ITEM_DTYPE)
        self.code_bytes, self.nblocks, self.small_numel = code, blocks, small
        if len(numels) >= 2 ** 31 or self.items.size >= 2 ** 31:
            raise ValueError("AdamW8bit: too many tensors or items for the 32-bit tables")

    @property
    def state_bytes(self) -> int:
        """Bytes of optimizer state: two code arrays, two absmax arrays and the fp32 m / v of the small tensors."""
        return 2 * self.code_bytes + 2 * 4 * self.nblocks + 2 * 4 * self.small_numel

    def bytes_per_step(self) -> int:
        """Bytes the kernel moves through memory per step, counted from its walk: per element of an 8-bit tensor it reads p, g and
        two codes and writes p and two codes (16 B); per block it reads and writes two scales (16 B); per element of a 32-bit
        tensor it reads p, g, m, v and writes p, m, v (28 B).  The tables, maps and hyper rows are a few bytes per item."""
        t = self.tensors
        n8 = int(t["numel"][t["mode"] == MODE_8BIT].sum())
        n32 = int(t["numel"][t["mode"] == MODE_32BIT].sum())
        return 16 * n8 + 16 * self.nblocks + 28 * n32
