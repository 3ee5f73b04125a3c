"""Small-M (weight-streaming) layers, cold vs L2-warm weights, row-major vs k-block-major weight operands.

Every case is captured REPS times into one CUDA graph; `cold` cycles over NW distinct weight packs (NW x weights >> 50 MB L2, the
regime of the real step where each layer's weights are read once per pass), `warm` reuses one pack.

  python tools/probe_smallm.py            -> table
  HCP_PROBE_ONE=conv8 python tools/probe_smallm.py   (one eager launch between cudaProfilerStart/Stop, for ncu)
"""
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import hcp_diffusion_b200.models  # noqa: E402,F401
from hcp_diffusion_b200 import ops  # noqa: E402
from hcp_diffusion_b200.ops import ConvPack, LinearPack  # noqa: E402

DEV, BF = "cuda", torch.bfloat16
REPS = 24


def rnd(*shape, scale=1.0):
    return torch.randn(*shape, device=DEV) * scale


def timed(fns):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for f in fns:
            f()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(REPS):
            fns[i % len(fns)]()
    best = 1e9
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1) * 1e3 / REPS)
    return best


def conv_case(B, H, Cin, Cout, tiled, nw):
    packs = []
    for _ in range(nw):
        p = ConvPack(rnd(Cout, Cin, 3, 3, scale=1 / math.sqrt(9 * Cin)), rnd(Cout, scale=0.1), 1)
        if tiled:
            p.tile_weights()
        packs.append(p)
    xs = [rnd(B, H * H, Cin).to(BF) for _ in range(4)]
    with torch.no_grad():
        return timed([(lambda i=i: ops.conv3x3(packs[i % nw], xs[i % 4], (B, H, H))) for i in range(max(nw, 4))])


def gemm_case(M, K, N, tiled, nw):
    packs = []
    for _ in range(nw):
        p = LinearPack(rnd(N, K, scale=1 / math.sqrt(K)), rnd(N, scale=0.1))
        if tiled:
            p.tile_weights()
        packs.append(p)
    xs = [rnd(M, K).to(BF) for _ in range(4)]
    with torch.no_grad():
        return timed([(lambda i=i: ops.fused_linear(packs[i % nw], [xs[i % 4]])) for i in range(max(nw, 4))])


one = os.environ.get("HCP_PROBE_ONE")
if one:
    tiled = os.environ.get("HCP_PROBE_TILED", "0") == "1"
    p = ConvPack(rnd(1280, 1280, 3, 3, scale=0.01), rnd(1280, scale=0.1), 1)
    if tiled:
        p.tile_weights()
    x = rnd(4, 64, 1280).to(BF)
    with torch.no_grad():
        for _ in range(2):
            ops.conv3x3(p, x, (4, 8, 8))
        torch.cuda.synchronize()
        torch.cuda.profiler.start()
        ops.conv3x3(p, x, (4, 8, 8))
        torch.cuda.synchronize()
        torch.cuda.profiler.stop()
    sys.exit(0)

print(f"{'case':44s} {'rowmajor warm':>14s} {'rowmajor cold':>14s} {'kblock warm':>12s} {'kblock cold':>12s}   (us per launch)")
for name, fn, args, wbytes in [
    ("conv3x3 B4 8x8 1280->1280", conv_case, (4, 8, 1280, 1280), 1280 * 1280 * 18),
    ("conv3x3 B4 8x8 2560->1280", conv_case, (4, 8, 2560, 1280), 2560 * 1280 * 18),
    ("conv3x3 B4 16x16 1280->1280", conv_case, (4, 16, 1280, 1280), 1280 * 1280 * 18),
    ("conv3x3 B4 16x16 2560->1280", conv_case, (4, 16, 2560, 1280), 2560 * 1280 * 18),
    ("conv3x3 B4 32x32 640->640", conv_case, (4, 32, 640, 640), 640 * 640 * 18),
    ("conv3x3 B4 32x32 1280->640", conv_case, (4, 32, 1280, 640), 1280 * 640 * 18),
    ("linear M256 K1280 N1280", gemm_case, (256, 1280, 1280), 1280 * 1280 * 2),
    ("linear M256 K5120 N1280", gemm_case, (256, 5120, 1280), 5120 * 1280 * 2),
    ("linear M1024 K1280 N1280", gemm_case, (1024, 1280, 1280), 1280 * 1280 * 2),
    ("linear M1024 K5120 N1280", gemm_case, (1024, 5120, 1280), 5120 * 1280 * 2),
    ("linear M1024 K1280 N10240", gemm_case, (1024, 1280, 10240), 10240 * 1280 * 2),
]:
    nw = max(4, int(300e6 // wbytes) + 1)
    r = []
    for tiled in (False, True):
        r.append(fn(*args, tiled, 1))
        r.append(fn(*args, tiled, nw))
        torch.cuda.empty_cache()
    print(f"{name:44s} {r[0]:14.2f} {r[1]:14.2f} {r[2]:12.2f} {r[3]:12.2f}   weights {wbytes / 1e6:.1f} MB, hbm floor {wbytes / 6.5677e6:.1f} us", flush=True)
