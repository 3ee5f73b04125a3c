"""Host-side tooling around the measurements (CPU only): tools/join_launches.py must keep aligning the library's C-ABI calls with the
kernel names it launches, otherwise a profiled step can no longer be attributed to call shapes."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_join_launches_consumes_every_kernel_of_the_committed_launch_list(golden_dir):
    # a small call log in the format of tools/profile_step.py and an `ncu --csv --metrics gpu__time_duration.sum` launch list of the
    # kernels those calls launch: split-K GEMM + finalize, the four phase launches of the stride-2 dgrad, one attention backward
    # launch per 64-column slice (d = 160: three), the device-side AdamW pair, a torch kernel the join must skip
    shapes = os.path.join(golden_dir, "launch_join_calls.json")
    launches = os.path.join(golden_dir, "launch_join_ncu.csv")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "join_launches.py"), shapes, launches],
                         capture_output=True, text=True, check=True).stdout
    first = out.splitlines()[0].split()                      # "kernels consumed N of N"
    assert first[:2] == ["kernels", "consumed"] and first[2] == first[4] == "24", out[:200]
    lines = out.splitlines()
    assert lines[1] == "total us 2987"
    # the attention backward at d = 160 is its prep, three slice launches and the dQ conversion: 8 + 3 x 30 + 4 us
    assert any('"d": 160, "fn": "hcp_attn_bwd_bf16"' in l and "102.0 us" in l for l in lines)
    # the stride-2 dgrad convolution is four GEMM launches of 14 us
    assert any('"fn": "hcp_conv3x3_bf16", "mode": 1' in l and "56.0 us" in l for l in lines)
