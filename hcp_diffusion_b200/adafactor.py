"""Adafactor over the flat parameter buffer: option parsing, the state layout and the device tables of `hcp_adafactor_flat`.

The optimizer is `transformers.optimization.Adafactor` (the reference's cfgs/train/examples/FT_sdxl.yaml): per tensor of the
module's shape, a factored second moment over the last two dims (row [P, R] and column [P, C] EMAs of a [P, R, C] view) for every
tensor with two or more dims, an elementwise one for 1-D tensors, and an optional first moment (`beta1`).  The kernels
(csrc/optim.cu) walk the tensors in tiles; this module cuts them and lays out the state and scratch buffers.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence, Tuple

import numpy as np

# transformers.optimization.Adafactor.__init__ defaults
DEFAULTS = {"lr": None, "eps": (1e-30, 1e-3), "clip_threshold": 1.0, "decay_rate": -0.8, "beta1": None, "weight_decay": 0.0,
            "scale_parameter": True, "relative_step": True, "warmup_init": False}
FLAG_SCALE_PARAMETER, FLAG_RELATIVE_STEP, FLAG_WARMUP_INIT, FLAG_BETA1 = 1, 2, 4, 8

TILE = 256              # threads per CTA = columns of a tile; also the rows of a tile
ITEM_ELEMS = 1 << 16    # elements per tile when small slabs are packed side by side
SLABS_PER_FACTOR_ITEM = 2048

TENSOR_DTYPE = np.dtype([("offset", "<i8"), ("numel", "<i8"), ("P", "<i8"), ("R", "<i8"), ("C", "<i8"), ("row", "<i8"), ("col", "<i8"),
                         ("rowpart", "<i8"), ("colpart", "<i8"), ("rmean", "<i8"), ("factored", "<i4"), ("group", "<i4"),
                         ("nct", "<i4"), ("nrch", "<i4"), ("item0", "<i4"), ("nitems", "<i4")])
ITEM_DTYPE = np.dtype([(k, "<i4") for k in ("tensor", "p0", "p1", "c0", "c1", "r0", "r1", "mode")])


def check_options(kw: Optional[dict]) -> dict:
    """The constructor keys of transformers' Adafactor with its defaults and its two refusals."""
    kw = dict(kw or {})
    unknown = set(kw) - set(DEFAULTS)
    if unknown:
        raise TypeError(f"unknown Adafactor options {sorted(unknown)}")
    out = {**DEFAULTS, **kw}
    out["eps"] = tuple(float(e) for e in out["eps"])
    if out["lr"] is not None and out["relative_step"]:
        raise ValueError("Cannot combine manual `lr` and `relative_step=True` options")
    if out["warmup_init"] and not out["relative_step"]:
        raise ValueError("`warmup_init=True` requires `relative_step=True`")
    return out


def hyper_row(opts: dict, lr: Optional[float], weight_decay: float) -> List[float]:
    """The 8 device floats of one parameter group: {lr, eps1, eps2, clip_threshold, decay_rate, beta1, weight_decay, flags}."""
    flags = ((FLAG_SCALE_PARAMETER if opts["scale_parameter"] else 0) | (FLAG_RELATIVE_STEP if opts["relative_step"] else 0) |
             (FLAG_WARMUP_INIT if opts["warmup_init"] else 0) | (FLAG_BETA1 if opts["beta1"] is not None else 0))
    return [float(lr or 0.0), opts["eps"][0], opts["eps"][1], float(opts["clip_threshold"]), float(opts["decay_rate"]),
            float(opts["beta1"] or 0.0), float(weight_decay), float(flags)]


def factored_view(shape: Sequence[int]) -> Optional[Tuple[int, int, int]]:
    """(P, R, C) of a tensor Adafactor factors (two or more dims; the leading dims are a batch), else None."""
    if len(shape) < 2:
        return None
    return math.prod(shape[:-2]), int(shape[-2]), int(shape[-1])


def state_numel(shapes: Sequence[Sequence[int]]) -> int:
    """Second-moment elements Adafactor keeps for these parameter shapes (P*R + P*C factored, numel otherwise)."""
    n = 0
    for s in shapes:
        f = factored_view(s)
        n += f[0] * (f[1] + f[2]) if f else math.prod(s)
    return n


class Layout:
    """Tensor table, tile lists and buffer sizes for parameters of `shapes` at flat `offsets`, tensor i in parameter group
    `groups[i]`."""

    def __init__(self, shapes: Sequence[Sequence[int]], offsets: Sequence[int], groups: Sequence[int]):
        tens = np.zeros(len(shapes), dtype=TENSOR_DTYPE)
        items: List[np.ndarray] = []
        fitems: List[np.ndarray] = []
        nitems, state, work_tail = 0, 0, []
        for i, (shape, off, grp) in enumerate(zip(shapes, offsets, groups)):
            numel = math.prod(shape)
            f = factored_view(shape)
            t = tens[i]
            t["offset"], t["numel"], t["group"], t["rowpart"], t["colpart"], t["rmean"], t["col"] = off, numel, grp, -1, -1, -1, -1
            if f is None:
                P, R, C = 1, -(-numel // TILE), TILE
                t["row"] = state
                state += numel
                ctiles = [(0, TILE)]
            else:
                P, R, C = f
                t["row"], t["col"] = state, state + P * R
                state += P * (R + C)
                ctiles = [(c0, min(C, c0 + TILE)) for c0 in range(0, C, TILE)] if C > TILE // 2 else [(0, C)]
            t["P"], t["R"], t["C"], t["factored"] = P, R, C, int(f is not None)
            t["nct"], t["nrch"] = len(ctiles), -(-R // TILE)
            k = TILE // (ctiles[0][1] - ctiles[0][0])
            rows = min(R, TILE)
            pper = k * max(1, ITEM_ELEMS // (k * (ctiles[0][1] - ctiles[0][0]) * rows))
            r0 = np.arange(0, R, TILE)
            p0 = np.arange(0, P, pper)
            c0 = np.array([c[0] for c in ctiles])
            c1 = np.array([c[1] for c in ctiles])
            rr, cc, pp = np.meshgrid(np.arange(len(r0)), np.arange(len(ctiles)), np.arange(len(p0)), indexing="ij")
            it = np.zeros(rr.size, dtype=ITEM_DTYPE)
            it["tensor"] = i
            it["p0"], it["p1"] = p0[pp.ravel()], np.minimum(p0[pp.ravel()] + pper, P)
            it["c0"], it["c1"] = c0[cc.ravel()], c1[cc.ravel()]
            it["r0"], it["r1"] = r0[rr.ravel()], np.minimum(r0[rr.ravel()] + TILE, R)
            t["item0"], t["nitems"] = nitems, it.size
            nitems += it.size
            items.append(it)
            if f is not None:
                work_tail.append(("rmean", i, P))
                if t["nct"] > 1:
                    work_tail.append(("rowpart", i, P * R * int(t["nct"])))
                if t["nrch"] > 1:
                    work_tail.append(("colpart", i, int(t["nrch"]) * P * C))
                if R >= 32:
                    fi = np.zeros(P, dtype=ITEM_DTYPE)
                    fi["p0"] = np.arange(P)
                    fi["p1"] = fi["p0"] + 1
                else:
                    s0 = np.arange(0, P, SLABS_PER_FACTOR_ITEM)
                    fi = np.zeros(s0.size, dtype=ITEM_DTYPE)
                    fi["p0"], fi["p1"], fi["mode"] = s0, np.minimum(s0 + SLABS_PER_FACTOR_ITEM, P), 1
                fi["tensor"] = i
                fitems.append(fi)
        work = 2 * nitems
        for field, i, n in work_tail:
            tens[i][field] = work
            work += n
        self.tensors = tens
        self.items = np.concatenate(items)
        self.factor_items = np.concatenate(fitems) if fitems else np.zeros(0, dtype=ITEM_DTYPE)
        self.state_numel = state
        self.work_numel = work
        if self.items.size >= 2 ** 30 or max(int(tens["P"].max()), int(tens["R"].max())) >= 2 ** 31:
            raise ValueError("Adafactor: too many tiles or slabs for the 32-bit item table")

    def bytes_per_step(self, beta1_groups=()) -> int:
        """Bytes the four passes move through memory per step, counted from the tile walk (state and scratch included)."""
        t = self.tensors
        n = int(t["numel"].sum())
        fac = t["factored"] == 1
        rowst = int((t["P"][fac] * t["R"][fac]).sum())
        colst = int((t["P"][fac] * t["C"][fac]).sum())
        vst = int(t["numel"][~fac].sum())
        m = int(t["numel"][np.isin(t["group"], list(beta1_groups))].sum()) if len(beta1_groups) else 0
        # (a) read p, g; EMA read+write of row / col / v.  (b) read row.  (c) read g, row, rmean, col, v.
        # (d) read p, g, row, rmean, col, v, write p, read+write m.  Partial sums and rmean are small and not counted.
        return 4 * (2 * n + 2 * (rowst + colst + vst) + rowst + (n + rowst + colst + vst) + (3 * n + rowst + colst + vst) + 2 * m)

