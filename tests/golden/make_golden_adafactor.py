"""Writes tests/golden/ref_adafactor.pt from the real transformers.optimization.Adafactor (the optimizer of the reference's
cfgs/train/examples/FT_sdxl.yaml): for every case of tests/adafactor_ref.GOLDEN_CASES, the parameters and the optimizer state
of every golden shape after six steps.  Inputs are regenerated from their seed (adafactor_ref.golden_inputs).

  python tests/golden/make_golden_adafactor.py
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from transformers.optimization import Adafactor  # noqa: E402

import adafactor_ref as A  # noqa: E402


def main():
    out = {"shapes": A.GOLDEN_SHAPES, "steps": A.GOLDEN_STEPS, "cases": []}
    for case in A.GOLDEN_CASES:
        p0, grads = A.golden_inputs(case)
        params = [torch.nn.Parameter(p.clone()) for p in p0]
        opt = Adafactor(params, **case["opts"])
        for step_grads in grads:
            for p, g in zip(params, step_grads):
                p.grad = g.clone()
            opt.step()
        state = [{k: (v.clone() if torch.is_tensor(v) else v) for k, v in opt.state[p].items() if k != "RMS"} for p in params]
        out["cases"].append({"name": case["name"], "params": [p.detach().clone() for p in params], "state": state})
    torch.save(out, os.path.join(HERE, "ref_adafactor.pt"))


if __name__ == "__main__":
    main()
