#!/usr/bin/env python
"""IFRNet benchmark: IFRNet-S and IFRNet-L (seeded weights) on a synthetic 1080p clip resident in HBM, multiplier 2.

    python tools/bench_ifrnet.py [--variants S L] [--frames 33] [--h 1080] [--w 1920] [--steps 3] [--warmup 1]
                                 [--torch-pairs 4] [--no-torch] [--profile]

One step = every pair of the clip (frames - 1 interpolated frames) through IfrnetEngine.forward as the node calls it at
multiplier 2: resize factor t = 1/2, embt = 1.0 (the node's default scale_factor), one pair per library call, timed with
CUDA events.  Prints one JSON line per variant:
  value            interpolated frames/s (median step)
  tflops           whole-model TFLOP/s: oracle.ifrnet.ifrnet_macs (the convolutions' logical channels, no padding
                   channels: 57.36 / 400.02 GMAC per 1080p frame) x 2 / time; element-wise work is not counted
  torch_*          oracle/ifrnet.py's PyTorch restatement of the reference model on the same GPU (fp32, cuDNN, TF32
                   allowed as by PyTorch's defaults, one pair per call as the reference node runs it)
  card             name and power limit of the GPU the numbers come from
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

from oracle import ifrnet as OI  # noqa: E402
from oracle import rife46 as O  # noqa: E402


def card(index: int) -> dict:
    """name and power limit of the card the numbers come from (read only: nvidia-smi --query-gpu)"""
    info = {"name": torch.cuda.get_device_name(index), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return info


def kernel_group(name: str) -> str:
    for key, group in (("streamconv", "conv (streamconv)"), ("first_conv", "first conv"), ("s2d", "space-to-depth"),
                       ("dec_in", "decoder input (warps)"), ("dec4_in", "decoder input (warps)"),
                       ("dec_flow", "flow accumulate"), ("final", "final warp + merge"), ("prep", "mean + resize"),
                       ("frame_sums", "mean + resize"), ("mean", "mean + resize")):
        if key in name:
            return group
    return "other"


def bench_variant(a, variant, clip_nchw):
    from cfi_b200.engine import IfrnetEngine
    sd = OI.synthetic_state_dict(variant, 0)
    eng = IfrnetEngine(sd, device=0, dtype="float32")
    npairs = a.frames - 1
    out = torch.empty((npairs, 1, 3, a.h, a.w), dtype=torch.float32, device="cuda")
    t, embt = 0.5, 1.0

    def step():
        for i in range(npairs):
            eng.forward(clip_nchw[i:i + 1], clip_nchw[i + 1:i + 2], t, embt, out=out[i])

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
    macs = OI.ifrnet_macs(variant, a.h, a.w, t)
    res = dict(metric=f"ifrnet_{variant}_frames_per_s", value=round(npairs / tm, 2), unit="interpolated frames/s",
               size=[a.h, a.w], frames=a.frames, multiplier=2, step_s=[round(x, 4) for x in times],
               gmac_per_frame=round(macs / 1e9, 2), tflops=round(2 * macs * npairs / tm / 1e12, 1),
               launches_per_frame=None, out_finite=bool(torch.isfinite(out).all()), card=card(0))
    n0 = eng.launch_count()
    eng.forward(clip_nchw[0:1], clip_nchw[1:2], t, embt, out=out[0])
    res["launches_per_frame"] = eng.launch_count() - n0

    if not a.no_torch:
        torch.backends.cudnn.allow_tf32 = True  # PyTorch's default for convolutions, stated for the record
        sdc = {k: v.cuda() for k, v in sd.items()}
        with torch.no_grad():
            OI.forward(sdc, clip_nchw[0:1], clip_nchw[1:2], t, embt)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(a.torch_pairs):
                y = OI.forward(sdc, clip_nchw[i:i + 1], clip_nchw[i + 1:i + 2], t, embt)
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
                g = kernel_group(ev.key)
                groups[g] = groups.get(g, 0.0) + dev_us / 1e3
        res["profile_ms_per_step"] = {k: round(v, 2) for k, v in sorted(groups.items(), key=lambda kv: -kv[1])}
    eng.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variants", nargs="+", default=["S", "L"])
    ap.add_argument("--frames", type=int, default=33)
    ap.add_argument("--h", type=int, default=1080)
    ap.add_argument("--w", type=int, default=1920)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--torch-pairs", type=int, default=4)
    ap.add_argument("--no-torch", action="store_true")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ifrnet: no CUDA device")
    import __graft_entry__ as ge
    ge.load_package()
    clip = O.synthetic_clip(a.frames, a.h, a.w, seed=7).cuda().permute(0, 3, 1, 2).contiguous()
    for v in a.variants:
        print(json.dumps(bench_variant(a, v, clip)), flush=True)


if __name__ == "__main__":
    main()
