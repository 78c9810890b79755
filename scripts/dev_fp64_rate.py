"""dev: measured fp64 issue intervals (vector DFMA vs DMMA) on the GPU box.
usage: python scripts/dev_fp64_rate.py [max SM clock in MHz]  (nvidia-smi --query-gpu=clocks.max.sm)
With the clock, the m16n8k8 interval is also printed as the fp64 tensor ceiling of the whole GPU at that clock: the rate the
large Cholesky's trailing update (chol_syrk_dmma_kernel) is measured against."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bundler_sfm_b200 import _lib

lib = _lib.load_library()
mhz = float(sys.argv[1]) if len(sys.argv) > 1 else 0.0
for mode, name in ((0, "DFMA"), (1, "DMMA m8n8k4"), (2, "DMMA m16n8k8")):
    for warps in (1, 4, 8, 16):
        v = lib.bsfm_measure_fp64_issue_cycles(mode, warps, 4096)
        print(f"{name:12s} warps/CTA={warps:2d}: {v:7.2f} cycles per warp instruction per sub-partition", flush=True)
    if mode == 2 and v > 0:
        per_clk = 4 * 16 * 8 * 8 * 2 / v       # four sub-partitions, 2048 FLOP per m16n8k8
        line = f"DMMA m16n8k8 ceiling: {per_clk:.0f} fp64 FLOP/clk/SM"
        if mhz > 0:
            import torch
            sms = torch.cuda.get_device_properties(0).multi_processor_count
            line += f" = {per_clk * sms * mhz * 1e6 / 1e12:.1f} TFLOP/s on {sms} SMs at {mhz:.0f} MHz"
        print(line, flush=True)
