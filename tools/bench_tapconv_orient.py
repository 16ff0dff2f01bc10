#!/usr/bin/env python
"""Time every RIFE-4.6 layer that the tapconv plan runs channel-major (64 output channels on the wgmma M, the tile's
128 cells on N) against the same layer with cells on M (debug impl=2), at the 1080p geometry, in one process.

    python tools/bench_tapconv_orient.py [--batch 8] [--dtype float16] [--iters 15] [--json out.json]

Per layer the two orientations alternate launch by launch; every launch is timed with CUDA events after a 256 MB
write that flushes L2, and the median is reported.  TFLOP/s come from the layer's MACs per cell (vfi_rife46_layer_plan)
and HBM GB/s from the activations a launch must read and write once.  Both orientations' outputs are compared (max abs
difference).  The JSON records the card's name and power limit (read only: nvidia-smi --query-gpu)."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402
from oracle import rife46 as O  # noqa: E402

BLOCK_C = (192, 128, 96, 64)
IMPL_NAMES = {0: "channel_major", 2: "cell_major"}


def card(index: int) -> dict:
    info = {"name": torch.cuda.get_device_name(index), "power_limit_w": None, "max_sm_mhz": None}
    try:
        r = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
        pw, mhz = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
        info["power_limit_w"], info["max_sm_mhz"] = float(pw), float(mhz)
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--dtype", default="float16", choices=["float16", "bfloat16"])
    ap.add_argument("--iters", type=int, default=15, help="timed launches per orientation and layer (median)")
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    ge.load_package()
    from cfi_b200.engine import Rife46Engine
    eng = Rife46Engine(O.synthetic_state_dict(0), 0, a.dtype)
    tdt = torch.float16 if a.dtype == "float16" else torch.bfloat16
    B, Hp, Wp = a.batch, 1088, 1920
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    rows = []
    for blk, s in enumerate((8, 4, 2, 1)):
        c = BLOCK_C[blk]
        h, w = Hp // s // 4, Wp // s // 4
        for layer in range(1, 10):
            pl = eng.layer_plan(blk, layer)
            if not pl["cmajor"]:
                continue
            g = torch.Generator().manual_seed(10 * blk + layer)
            x = (0.1 * torch.randn(B, h, w, 2 * c if layer == 1 else c, generator=g)).to(tdt).cuda()
            outs = {i: torch.empty(B, h, w, c, dtype=tdt, device="cuda") for i in IMPL_NAMES}
            for _ in range(3):
                for i in IMPL_NAMES:
                    eng.debug_layer(blk, layer, x, outs[i], impl=i)
            torch.cuda.synchronize()
            diff = (outs[0].float() - outs[2].float()).abs().max().item()
            times = {i: [] for i in IMPL_NAMES}
            for _ in range(a.iters):
                for i in IMPL_NAMES:
                    flush.zero_()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    eng.debug_layer(blk, layer, x, outs[i], impl=i)
                    e1.record()
                    torch.cuda.synchronize()
                    times[i].append(e0.elapsed_time(e1))
            flops = 2.0 * pl["macs_per_cell"] * B * h * w
            hbm_bytes = x.numel() * x.element_size() + outs[0].numel() * outs[0].element_size()
            row = dict(block=blk, layer=layer, c=c, cin=x.shape[-1], grid=[h, w], batch=B, dtype=a.dtype,
                       n_cta=pl["n_cta"], stages=pl["stages"], flops=flops, hbm_bytes=hbm_bytes,
                       max_abs_diff=diff, bit_identical=diff == 0.0)
            for i, name in IMPL_NAMES.items():
                ms = statistics.median(times[i])
                row[name] = dict(ms=ms, tflops=flops / ms / 1e9, hbm_gbs=hbm_bytes / ms / 1e6)
            row["speedup"] = row["cell_major"]["ms"] / row["channel_major"]["ms"]
            rows.append(row)
            print(f"block {blk} layer {layer} ({x.shape[-1]}->{c}, {h}x{w}, batch {B}): "
                  f"channel-major {row['channel_major']['ms']:.4f} ms {row['channel_major']['tflops']:.0f} TFLOP/s "
                  f"{row['channel_major']['hbm_gbs']:.0f} GB/s | cell-major {row['cell_major']['ms']:.4f} ms "
                  f"{row['cell_major']['tflops']:.0f} TFLOP/s | x{row['speedup']:.3f} | max abs diff {diff:g}", flush=True)
    result = dict(card=card(torch.cuda.current_device()), how=f"CUDA events per launch after an L2 flush, median of "
                  f"{a.iters}, orientations alternated", layers=rows)
    print(json.dumps(result))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(result, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
