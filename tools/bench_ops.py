"""In-graph micro-benchmarks of the library's kernels at the shapes of the SD1.5 bs=4 step.

ncu launch lists (profiles/*launches*.csv) time every kernel cold and serialised; inside the captured step graph the operands of a
kernel were just written by its producer and sit in the 50 MB L2.  This script reproduces that regime: every op is captured
REPS times back to back into one CUDA graph, cycling over a small ring of buffers, and the graph replay is timed with CUDA events.

  python tools/bench_ops.py [filter-substring]      -> one line per op: us per launch, TF/s or GB/s (algorithmic bytes)
"""
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import hcp_diffusion_b200.models  # noqa: E402,F401  (models first: runtime <-> models import cycle)
from hcp_diffusion_b200 import ops  # noqa: E402
from hcp_diffusion_b200.ops import ConvPack, LinearPack, LoraBlockRef  # noqa: E402
from hcp_diffusion_b200.runtime import pack_lora  # noqa: E402

DEV = "cuda"
BF = torch.bfloat16
REPS, RING = 24, 4
FILTER = sys.argv[1] if len(sys.argv) > 1 else ""
rows = []


def bench(name, make, flops=None, bytes_=None):
    """make(i) -> callable running the op on buffer set i (i < RING)."""
    if FILTER and FILTER not in name:
        return
    fns = [make(i) for i in range(RING)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for f in fns:
            f()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for r in range(REPS):
            fns[r % RING]()
    for _ in range(2):
        g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = 1e9
    for _ in range(5):
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1) * 1e3 / REPS)
    extra = ""
    if flops:
        extra += f"  {flops / best * 1e-6:8.0f} TF/s"
    if bytes_:
        extra += f"  {bytes_ / best * 1e-3:8.0f} GB/s"
    line = f"{name:58s} {best:8.2f} us{extra}"
    print(line, flush=True)
    rows.append(line)


def rnd(*shape, scale=1.0):
    return (torch.randn(*shape, device=DEV) * scale)


def gemm_case(M, K, N, rank=0, res=False):
    W = rnd(N, K, scale=1 / math.sqrt(K))
    pack = LinearPack(W, rnd(N, scale=0.1))
    if rank:
        pack.attach_lora([LoraBlockRef(rnd(rank, K, scale=0.05), rnd(N, rank, scale=0.05), 0.125, 0)])

        class G:
            pass
        g = G()
        g.pack = pack
        pack_lora([g])
    xs = [rnd(M, K).to(BF) for _ in range(RING)]
    rs = [rnd(M, N).to(BF) for _ in range(RING)] if res else [None] * RING

    def make(i):
        return lambda: ops.fused_linear(pack, [xs[i]], rs[i])
    with torch.no_grad():
        bench(f"linear M{M} K{K} N{N}" + (f" +lora r{rank}" if rank else "") + (" +res" if res else ""), make, flops=2.0 * M * N * K)


def conv_case(B, H, Cin, Cout, stride=1):
    pack = ConvPack(rnd(Cout, Cin, 3, 3, scale=1 / math.sqrt(9 * Cin)), rnd(Cout, scale=0.1), stride)
    xs = [rnd(B, H * H, Cin).to(BF) for _ in range(RING)]

    def make(i):
        return lambda: ops.conv3x3(pack, xs[i], (B, H, H))
    with torch.no_grad():
        bench(f"conv3x3 B{B} {H}x{H} {Cin}->{Cout} s{stride}", make, flops=2.0 * B * (H // stride) ** 2 * Cout * 9 * Cin)


def gn_case(B, HW, C, bwd):
    gamma, beta = 1 + 0.1 * rnd(C), 0.1 * rnd(C)
    xs = [rnd(B, HW, C).to(BF).requires_grad_(bwd) for _ in range(RING)]
    dy = rnd(B, HW, C).to(BF)
    n = B * HW * C * 2

    def make(i):
        if not bwd:
            return lambda: ops.group_norm(gamma, beta, 32, 1e-5, True, xs[i])
        def f():
            xs[i].grad = None
            ops.group_norm(gamma, beta, 32, 1e-5, True, xs[i])[0].backward(dy)
        return f
    if bwd:
        bench(f"groupnorm fwd+bwd B{B} HW{HW} C{C}", make, bytes_=5 * n)
    else:
        with torch.no_grad():
            bench(f"groupnorm fwd B{B} HW{HW} C{C}", make, bytes_=2 * n)


def ln_case(M, C, bwd):
    gamma, beta = 1 + 0.1 * rnd(C), 0.1 * rnd(C)
    xs = [rnd(M, C).to(BF).requires_grad_(bwd) for _ in range(RING)]
    dy = rnd(M, C).to(BF)
    n = M * C * 2

    def make(i):
        if not bwd:
            return lambda: ops.layer_norm(gamma, beta, 1e-5, xs[i])
        def f():
            xs[i].grad = None
            ops.layer_norm(gamma, beta, 1e-5, xs[i])[0].backward(dy)
        return f
    if bwd:
        bench(f"layernorm fwd+bwd M{M} C{C}", make, bytes_=5 * n)
    else:
        with torch.no_grad():
            bench(f"layernorm fwd M{M} C{C}", make, bytes_=2 * n)


def attn_case(B, H, Lq, Lkv, d, bwd):
    C = H * d
    if Lq == Lkv:
        srcs = [rnd(B, Lq, 3 * C).to(BF).requires_grad_(bwd) for _ in range(RING)]
        kvs = [None] * RING
        offs = (0, C, 2 * C)
    else:
        srcs = [rnd(B, Lq, C).to(BF).requires_grad_(bwd) for _ in range(RING)]
        kvs = [rnd(B, Lkv, 2 * C).to(BF).requires_grad_(bwd) for _ in range(RING)]
        offs = (0, 0, C)
    do = rnd(B, Lq, C).to(BF)
    fl = 4.0 * B * H * Lq * Lkv * d

    def make(i):
        if not bwd:
            return lambda: ops.attention(H, C, offs, srcs[i], kvs[i])
        def f():
            srcs[i].grad = None
            if kvs[i] is not None:
                kvs[i].grad = None
            ops.attention(H, C, offs, srcs[i], kvs[i]).backward(do)
        return f
    if bwd:
        bench(f"attention fwd+bwd B{B} H{H} Lq{Lq} Lkv{Lkv} d{d}", make, flops=3.5 * fl)
    else:
        with torch.no_grad():
            bench(f"attention fwd B{B} H{H} Lq{Lq} Lkv{Lkv} d{d}", make, flops=fl)


def geglu_case(M, F_):
    us = [rnd(M, 2 * F_).to(BF) for _ in range(RING)]

    def make(i):
        return lambda: ops.GegluFn.apply(us[i])
    with torch.no_grad():
        bench(f"geglu fwd M{M} F{F_}", make, bytes_=M * F_ * 2 * 3)


def linear_bwd_case(M, K, N, rank):
    W = rnd(N, K, scale=1 / math.sqrt(K))
    pack = LinearPack(W, None)
    down, up = rnd(rank, K, scale=0.05).requires_grad_(True), rnd(N, rank, scale=0.05).requires_grad_(True)
    pack.attach_lora([LoraBlockRef(down, up, 0.125, 0)])

    class G:
        pass
    g = G()
    g.pack = pack
    pack_lora([g])
    xs = [rnd(M, K).to(BF).requires_grad_(True) for _ in range(RING)]
    dy = rnd(M, N).to(BF)

    def make(i):
        def f():
            xs[i].grad = None
            ops.fused_linear(pack, [xs[i]], None).backward(dy)
        return f
    bench(f"linear+lora fwd+bwd (5 GEMMs + grad kernel) M{M} K{K} N{N} r{rank}", make, flops=4.0 * M * N * K)


def tiny_case():
    """Launch floor: a 1-CTA elementwise kernel, back to back in the graph."""
    from hcp_diffusion_b200._lib import call, stream_ptr
    a, b, o = (torch.zeros(64, device=DEV, dtype=BF) for _ in range(3))

    def make(i):
        return lambda: call("hcp_add_bf16", a.data_ptr(), b.data_ptr(), 64, o.data_ptr(), stream_ptr())
    bench("tiny kernel (add_bf16 on 64 elements): graph launch floor", make)


if __name__ == "__main__":
    torch.manual_seed(0)
    B = 4
    tiny_case()
    gemm_case(16384, 320, 320, res=True)
    gemm_case(16384, 320, 320, rank=8)
    for M, K, N in [(16384, 320, 320), (4096, 640, 640), (1024, 1280, 1280), (256, 1280, 1280), (16384, 320, 64), (4096, 640, 64), (1024, 1280, 64),
                    (16384, 320, 2560), (16384, 1280, 320), (16384, 2560, 320), (4096, 640, 5120), (1024, 1280, 10240), (1024, 5120, 1280),
                    (1024, 10240, 1280)]:
        gemm_case(M, K, N)
    gemm_case(16384, 320, 320, rank=8, res=True)
    gemm_case(16384, 320, 960, rank=24)
    gemm_case(1024, 1280, 1280, rank=8, res=True)
    linear_bwd_case(16384, 320, 320, 8)
    linear_bwd_case(1024, 1280, 1280, 8)
    for H, Cin, Cout in [(64, 320, 320), (64, 640, 320), (64, 960, 320), (32, 640, 640), (32, 1280, 640), (16, 1280, 1280), (16, 2560, 1280), (8, 1280, 1280),
                         (8, 2560, 1280)]:
        conv_case(B, H, Cin, Cout)
    conv_case(B, 64, 320, 320, stride=2)
    for HW, C in [(4096, 320), (4096, 640), (1024, 640), (256, 1280), (64, 1280), (64, 2560)]:
        gn_case(B, HW, C, False)
        gn_case(B, HW, C, True)
    for M, C in [(16384, 320), (4096, 640), (1024, 1280)]:
        ln_case(M, C, False)
        ln_case(M, C, True)
    for Lq, Lkv, d in [(4096, 4096, 40), (4096, 77, 40), (1024, 1024, 80), (1024, 77, 80), (256, 256, 160), (256, 77, 160)]:
        attn_case(B, 8, Lq, Lkv, d, False)
        attn_case(B, 8, Lq, Lkv, d, True)
    geglu_case(16384, 1280)
    os.makedirs("gpurun_out", exist_ok=True)
    open("gpurun_out/bench_ops.txt", "w").write("\n".join(rows) + "\n")
