"""The optimizer pass alone on one GPU: hcp_adamw_flat_dev, hcp_lion_flat_dev, hcp_adamw8bit_flat and hcp_prodigy_flat over flat
fp32 buffers of a whole UNet, each captured in a CUDA graph and timed alternately in one process (CUDA events around `--reps` replays, `--rounds`
rounds, median).  AdamW8bit walks a table that cuts the buffer like a UNet: 1280 x 1280 weights (8-bit) each followed by a
1280-element bias (fp32 moments), the remainder one more 8-bit tensor.

Traffic is counted from the kernels: AdamW reads p, g, m, v and writes p, m, v (28 B per parameter); Lion reads p, g, m and writes
p, m (20 B); AdamW8bit is adamw8bit.Layout.bytes_per_step (16 B per 8-bit parameter plus 16 B per 256-element block, 28 B per
parameter of the biases); Prodigy reads p, g, p0, s, m, v and writes s, m, v, then reads p, m, v and writes p (52 B, one
segment; its fp64 scalars and per-CTA partials are a few kB).  The step counter, the hyper row and the clip's sum of squares are a few bytes.  Prints one JSON line per size with
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

from hcp_diffusion_b200 import adamw8bit, prodigy  # noqa: E402
from hcp_diffusion_b200._lib import call, stream_ptr  # noqa: E402

SD15, SDXL = 859_520_964, 2_567_463_684          # trainable parameters of the SD1.5 and SDXL-base UNets
BYTES = {"adamw": 28, "lion": 20, "prodigy": 52}
W, B = 1280 * 1280, 1280


def unet_like_layout(n):
    """adamw8bit.Layout of weights of W elements each followed by a bias of B, the rest one more weight (16-byte aligned offsets)."""
    numels = []
    while sum(numels) + W + B <= n:
        numels += [W, B]
    if n - sum(numels) > 0:
        numels.append(n - sum(numels))
    offsets, off = [], 0
    for k in numels:
        offsets.append(off)
        off += (k + 3) // 4 * 4
    return adamw8bit.Layout(numels, offsets, [0] * len(numels)), off
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
    lay, nflat = unet_like_layout(n)
    assert nflat <= n4
    codes = torch.zeros(2 * lay.code_bytes, dtype=torch.uint8, device="cuda")
    absmax = torch.zeros(2 * lay.nblocks, device="cuda")
    state32 = torch.zeros(max(2 * lay.small_numel, 4), device="cuda")
    maps = adamw8bit.maps().cuda()
    to_dev = lambda a: torch.from_numpy(a.view("uint8").copy()).cuda()  # noqa: E731
    tens_d, items_d = to_dev(lay.tensors), to_dev(lay.items)
    hyper8 = torch.tensor([[1e-6, 0.9, 0.999, 1e-8, 1e-2]], device="cuda")
    steps8 = torch.zeros(1, dtype=torch.int32, device="cuda")
    BYTES["adamw8bit"] = lay.bytes_per_step() / n
    p0, s = torch.zeros_like(p), torch.zeros_like(p)
    pd_segs = prodigy.segment_table([(0, n, 1.0, 1e-2)])
    pd_segs_d = torch.from_numpy(pd_segs.view("int64").copy()).cuda()
    pd_hyper = torch.tensor(prodigy.hyper_row(prodigy.check_options({"use_bias_correction": True}), 0.9, 0.999, 1e-8),
                            dtype=torch.float64, device="cuda")
    pd_state = torch.tensor(prodigy.initial_state(1e-6), dtype=torch.float64, device="cuda")
    pd_work = torch.zeros(prodigy.WORKSPACE_BYTES // 8, dtype=torch.float64, device="cuda")
    graphs = {
        "adamw": graph_of(lambda: call("hcp_adamw_flat_dev", p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), n,
                                       hyper["adamw"].data_ptr(), *tail())),
        "lion": graph_of(lambda: call("hcp_lion_flat_dev", p.data_ptr(), g.data_ptr(), m.data_ptr(), n, hyper["lion"].data_ptr(), *tail())),
        "adamw8bit": graph_of(lambda: call("hcp_adamw8bit_flat", p.data_ptr(), g.data_ptr(), codes.data_ptr(), absmax.data_ptr(),
                                           state32.data_ptr(), maps.data_ptr(), lay.tensors.ctypes.data, tens_d.data_ptr(),
                                           len(lay.tensors), lay.items.ctypes.data, items_d.data_ptr(), lay.items.size, nflat,
                                           lay.code_bytes, lay.nblocks, lay.small_numel, hyper8.data_ptr(), steps8.data_ptr(), 1, 1.0,
                                           sumsq.data_ptr(), 1.0, stream_ptr())),
        "prodigy": graph_of(lambda: call("hcp_prodigy_flat", p.data_ptr(), g.data_ptr(), p0.data_ptr(), s.data_ptr(), m.data_ptr(),
                                         v.data_ptr(), n, pd_segs.ctypes.data, pd_segs_d.data_ptr(), 1, pd_hyper.data_ptr(),
                                         pd_state.data_ptr(), pd_work.data_ptr(), prodigy.WORKSPACE_BYTES, 1.0, sumsq.data_ptr(), 1.0,
                                         step.data_ptr(), stream_ptr())),
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
        out[name] = {"ms": round(ms, 3), "ms_min": round(min(ts), 3), "ms_max": round(max(ts), 3), "bytes_per_param": round(BYTES[name], 3),
                     "GB_s": round(gbs, 1), "share_of_3.35TBs": round(gbs / (HBM_TBS * 1e3), 3)}
    print(json.dumps(out), flush=True)
    del p, g, m, v, p0, s, codes, absmax, state32, graphs
    torch.cuda.empty_cache()
