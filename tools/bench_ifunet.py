#!/usr/bin/env python
"""IFUnet benchmark: IFUNetModel (seeded weights) on a synthetic 1080p clip resident in HBM, multiplier 2, scale_factor
1.0, with `ensemble` on (the node's default) or off.

    python tools/bench_ifunet.py [--frames 9] [--h 1080] [--w 1920] [--steps 3] [--warmup 1] [--no-ensemble]
                                 [--torch-pairs 2] [--no-torch] [--profile]

One step = every pair of the clip (frames - 1 interpolated frames) through IfunetEngine.forward as the node calls it, one
pair per library call at t = 0.5, timed with CUDA events.  Prints one JSON line:
  value            interpolated frames/s (median step); step_s holds every step
  tflops           whole-model TFLOP/s: oracle.ifunet.ifunet_macs (1438.4 / 1755.3 GMAC per 1080p frame without / with
                   ensemble: the logical channels, not the padded ones) x 2 / time; element-wise work is not counted
  torch_*          oracle/ifunet.py's PyTorch restatement of the reference model on the same GPU (fp32, cuDNN, TF32 allowed,
                   one pair per call as the reference node runs it), and the largest difference on the last frame
  launches_per_frame  kernel launches of one library call
  card             name, power limit and maximum SM clock of the GPU, read in the same call
  profile          (--profile) device time per kernel group of one step, from torch.profiler in a separate run
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ifunet as OU  # noqa: E402
from oracle import rife46 as O  # noqa: E402


def card(index: int) -> dict:
    """name, power limit and maximum SM clock of the card the numbers come from (read only: nvidia-smi --query-gpu)"""
    info = {"name": torch.cuda.get_device_name(index), "power_limit_w": None, "max_sm_clock_mhz": None}
    try:
        r = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
        pw, clk = r.stdout.strip().splitlines()[0].split(",")
        info["power_limit_w"] = float(pw)
        info["max_sm_clock_mhz"] = float(clk)
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return info


GROUPS = (("streamconv", "streamconv"), ("ifu_pool", "cbam"), ("ifu_gate", "cbam"), ("ifu_compress", "cbam"),
          ("ifu_spatial", "cbam"), ("ifu_convex", "convex + flow update"), ("ifu_flow_update", "convex + flow update"),
          ("ifu_stem", "stems"), ("ifu_s2d", "space-to-depth / phases"), ("ifu_d2s", "space-to-depth / phases"),
          ("nearest16", "nearest x2"), ("ifu_add", "residual adds"), ("ifu_rrdb_res", "residual adds"),
          ("ifu_fb_", "flowblock in / out + warps"), ("ifu_warp", "flowblock in / out + warps"),
          ("ifu_flow_in", "inputs"), ("ifu_fusion_in", "inputs"), ("ifu_ctx_warp", "context"), ("ifu_merge", "final"),
          ("ifu_final", "final"), ("Memset", "memset"))


def kernel_group(name: str) -> str:
    for key, group in GROUPS:
        if key in name:
            return group
    return "other"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=9)
    ap.add_argument("--h", type=int, default=1080)
    ap.add_argument("--w", type=int, default=1920)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--torch-pairs", type=int, default=2)
    ap.add_argument("--no-ensemble", action="store_true")
    ap.add_argument("--no-torch", action="store_true")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ifunet: no CUDA device")
    import __graft_entry__ as ge
    ge.load_package()
    from cfi_b200.engine import IfunetEngine
    clip = O.synthetic_clip(a.frames, a.h, a.w, seed=7).cuda().permute(0, 3, 1, 2).contiguous()
    sd = OU.synthetic_state_dict(0)
    eng = IfunetEngine(sd, device=0, dtype="float32")
    ens = not a.no_ensemble
    npairs = a.frames - 1
    out = torch.empty((npairs, 1, 3, a.h, a.w), dtype=torch.float32, device="cuda")

    def step():
        for i in range(npairs):
            eng.forward(clip[i:i + 1], clip[i + 1:i + 2], 0.5, 1.0, ens, out=out[i])

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    times = []
    for _ in range(a.steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        step()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3)
    tm = statistics.median(times)
    macs = OU.ifunet_macs(a.h, a.w, 1.0, ens)
    res = dict(metric="ifunet_frames_per_s", value=round(npairs / tm, 2), unit="interpolated frames/s", size=[a.h, a.w],
               frames=a.frames, multiplier=2, scale_factor=1.0, ensemble=ens, step_s=[round(x, 4) for x in times],
               gmac_per_frame=round(macs / 1e9, 1), tflops=round(2 * macs * npairs / tm / 1e12, 1),
               launches_per_frame=None, out_finite=bool(torch.isfinite(out).all()))
    n0 = eng.launch_count()
    eng.forward(clip[0:1], clip[1:2], 0.5, 1.0, ens, out=out[0])
    torch.cuda.synchronize()
    res["launches_per_frame"] = eng.launch_count() - n0

    if not a.no_torch:
        torch.backends.cudnn.allow_tf32 = True  # PyTorch's default for convolutions, stated for the record
        sdc = {k: v.cuda() for k, v in sd.items()}
        with torch.no_grad():
            OU.forward(sdc, clip[0:1], clip[1:2], 0.5, 1.0, ens)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(a.torch_pairs):
                y = OU.forward(sdc, clip[i:i + 1], clip[i + 1:i + 2], 0.5, 1.0, ens)
            e1.record()
            torch.cuda.synchronize()
        tt = e0.elapsed_time(e1) / 1e3 / a.torch_pairs
        diff = float((y - out[a.torch_pairs - 1]).abs().max())
        res.update(torch_frames_per_s=round(1 / tt, 2), speedup_vs_torch=round(npairs / tm * tt, 2),
                   max_abs_diff_vs_torch=round(diff, 5))
        del sdc

    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step()
            torch.cuda.synchronize()
        groups = {}
        for ev in prof.key_averages():
            dev_us = getattr(ev, "device_time_total", None)
            if dev_us is None:
                dev_us = getattr(ev, "cuda_time_total", 0)
            if dev_us:
                k = kernel_group(ev.key)
                groups[k] = groups.get(k, 0.0) + dev_us / 1e3
        total = sum(groups.values())
        res["profile_ms_per_step"] = {k: round(v, 2) for k, v in sorted(groups.items(), key=lambda kv: -kv[1])}
        res["profile_share"] = {k: round(v / total, 3) for k, v in sorted(groups.items(), key=lambda kv: -kv[1])}
    res["card"] = card(0)
    eng.close()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
