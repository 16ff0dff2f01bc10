#!/usr/bin/env python
"""CAIN benchmark: CAIN(depth=3) (seeded weights) on a synthetic 1080p clip resident in HBM, multiplier 2.

    python tools/bench_cain.py [--frames 17] [--h 1080] [--w 1920] [--steps 3] [--warmup 1] [--torch-pairs 3]
                               [--no-torch] [--profile]

One step = every pair of the clip (frames - 1 interpolated frames) through CainEngine.forward as the node calls it, one
pair per library call, timed with CUDA events.  Prints one JSON line:
  value            interpolated frames/s (median step)
  tflops           whole-model TFLOP/s: oracle.cain.cain_macs (1467.67 GMAC per 1080p frame: the convolutions on the
                   h x w trunk grid, not the bordered one they run on) x 2 / time; element-wise work is not counted
  tiles            16 x 8 tiles of one conv on the bordered (h + 2) x (w + 2) grid and on the h x w grid it stands for
  torch_*          oracle/cain.py's PyTorch restatement of the reference model on the same GPU (fp32, cuDNN, TF32 allowed,
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

from oracle import cain as OC  # noqa: E402
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


GROUPS = (("streamconv", "streamconv"), ("cain_chan_sums", "attention sums + gate"), ("cain_gate", "attention sums + gate"),
          ("cain_apply", "apply + border"), ("cain_border", "apply + border"), ("cain_frame_sums", "prep"),
          ("cain_prep", "prep"), ("cain_final", "final"))


def kernel_group(name: str) -> str:
    for key, group in GROUPS:
        if key in name:
            return group
    return "other"


def tiles(h, w):
    return ((h + 15) // 16) * ((w + 7) // 8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=17)
    ap.add_argument("--h", type=int, default=1080)
    ap.add_argument("--w", type=int, default=1920)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--torch-pairs", type=int, default=3)
    ap.add_argument("--no-torch", action="store_true")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cain: no CUDA device")
    import __graft_entry__ as ge
    ge.load_package()
    from cfi_b200.engine import CainEngine
    clip = O.synthetic_clip(a.frames, a.h, a.w, seed=7).cuda().permute(0, 3, 1, 2).contiguous()
    sd = OC.synthetic_state_dict(0)
    eng = CainEngine(sd, device=0, dtype="float32")
    npairs = a.frames - 1
    out = torch.empty((npairs, 1, 3, a.h, a.w), dtype=torch.float32, device="cuda")

    def step():
        for i in range(npairs):
            eng.forward(clip[i:i + 1], clip[i + 1:i + 2], out=out[i])

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
    macs = OC.cain_macs(a.h, a.w)
    g = OC.geometry(a.h, a.w)
    res = dict(metric="cain_frames_per_s", value=round(npairs / tm, 2), unit="interpolated frames/s", size=[a.h, a.w],
               frames=a.frames, multiplier=2, step_s=[round(x, 4) for x in times], gmac_per_frame=round(macs / 1e9, 2),
               tflops=round(2 * macs * npairs / tm / 1e12, 1),
               tiles=dict(bordered=tiles(g["gh"] + 2, g["gw"] + 2), grid=tiles(g["gh"], g["gw"]),
                          sms=torch.cuda.get_device_properties(0).multi_processor_count),
               launches_per_frame=None, out_finite=bool(torch.isfinite(out).all()))
    n0 = eng.launch_count()
    eng.forward(clip[0:1], clip[1:2], out=out[0])
    torch.cuda.synchronize()
    res["launches_per_frame"] = eng.launch_count() - n0

    if not a.no_torch:
        torch.backends.cudnn.allow_tf32 = True  # PyTorch's default for convolutions, stated for the record
        sdc = {k: v.cuda() for k, v in sd.items()}
        with torch.no_grad():
            OC.forward(sdc, clip[0:1], clip[1:2])
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(a.torch_pairs):
                y = OC.forward(sdc, clip[i:i + 1], clip[i + 1:i + 2])
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
