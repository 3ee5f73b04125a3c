"""The optimizer pass alone on one GPU: hcp_adamw_flat_dev and hcp_lion_flat_dev over flat fp32 buffers of a whole UNet, each
captured in a CUDA graph and timed alternately in one process (CUDA events around `--reps` replays, `--rounds` rounds, median).

Traffic is counted from the kernels: AdamW reads p, g, m, v and writes p, m, v (28 B per parameter); Lion reads p, g, m and writes
p, m (20 B).  The step counter, the hyper row and the clip's sum of squares are a few bytes.  Prints one JSON line per size with
ms, achieved GB/s and the share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), plus the card name and power limit.

  python tools/bench_optim.py [--sizes 859520964 2567463684] [--reps 5] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from hcp_diffusion_b200._lib import call, stream_ptr  # noqa: E402

SD15, SDXL = 859_520_964, 2_567_463_684          # trainable parameters of the SD1.5 and SDXL-base UNets
BYTES = {"adamw": 28, "lion": 20}
HBM_TBS = 3.35

ap = argparse.ArgumentParser()
ap.add_argument("--sizes", type=int, nargs="+", default=[SD15, SDXL])
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--rounds", type=int, default=5)
args = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_optim.py measures on a GPU; none is visible")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def graph_of(fn):
    fn()                                          # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


for n in args.sizes:
    n4 = (n + 3) // 4 * 4
    gen = torch.Generator(device="cuda").manual_seed(0)
    p = torch.randn(n4, device="cuda", generator=gen)
    g = torch.randn(n4, device="cuda", generator=gen).mul_(1e-3)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    hyper = {"adamw": torch.tensor([1e-6, 0.9, 0.999, 1e-8, 1e-2], device="cuda"),
             "lion": torch.tensor([1e-7, 0.9, 0.99, 1e-8, 1e-2], device="cuda")}
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    sumsq = torch.zeros(1, device="cuda")
    call("hcp_sumsq", g.data_ptr(), n, sumsq.data_ptr(), stream_ptr())
    tail = lambda: (1.0, sumsq.data_ptr(), 1.0, step.data_ptr(), stream_ptr())  # noqa: E731
    graphs = {
        "adamw": graph_of(lambda: call("hcp_adamw_flat_dev", p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), n,
                                       hyper["adamw"].data_ptr(), *tail())),
        "lion": graph_of(lambda: call("hcp_lion_flat_dev", p.data_ptr(), g.data_ptr(), m.data_ptr(), n, hyper["lion"].data_ptr(), *tail())),
    }
    times = {k: [] for k in graphs}
    for _ in range(args.rounds):
        for name, gr in graphs.items():
            gr.replay()                           # one untimed replay after switching
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                gr.replay()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.reps)
    assert bool(torch.isfinite(p[:1 << 20]).all())
    out = {"params": n, "gpu": card()}
    for name, ts in times.items():
        ms = statistics.median(ts)
        gbs = BYTES[name] * n / (ms * 1e-3) / 1e9
        out[name] = {"ms": round(ms, 3), "ms_min": round(min(ts), 3), "ms_max": round(max(ts), 3), "bytes_per_param": BYTES[name],
                     "GB_s": round(gbs, 1), "share_of_3.35TBs": round(gbs / (HBM_TBS * 1e3), 3)}
    print(json.dumps(out), flush=True)
    del p, g, m, v, graphs
    torch.cuda.empty_cache()
