#!/usr/bin/env python
"""FLAVR benchmark: the FLAVR_2x.pth model (seeded weights) on a synthetic 1080p clip resident in HBM.

    python tools/bench_flavr.py [--frames 64] [--h 1080] [--w 1920] [--windows 4] [--steps 3] [--warmup 1]
                                [--torch-windows 4] [--no-torch] [--profile]

One step = every 4-frame window of the clip (frames - 3 interpolated frames) through FlavrEngine.forward, `--windows`
windows per library call, timed with CUDA events.  Prints one JSON line:
  value            interpolated frames/s (median step)
  tflops           whole-model TFLOP/s: the MACs of the model's layer shapes at the padded size (computed below,
                   16.96 TFLOP per 1080p frame) x 2 / time; gates, means and element-wise work are not counted
  torch_*          oracle/flavr.py's PyTorch restatement of the reference model on the same GPU (fp32, cuDNN, TF32
                   allowed as by PyTorch's defaults, one window per call as the reference node runs it)
  card             name and power limit of the GPU the numbers come from
  profile          (--profile) device time per kernel group of one step, from torch.profiler in a separate run
The clip generator is SURVEY.md's config-2 one (oracle.rife46.synthetic_clip).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import flavr as OV  # noqa: E402
from oracle import rife46 as O  # noqa: E402


def flavr_macs(hp: int, wp: int) -> int:
    """Multiply-accumulates of one window (4 planes) at the padded size hp x wp, from the layer shapes."""
    T = 4
    p2, p4, p8, pp = (hp // 2) * (wp // 2), (hp // 4) * (wp // 4), (hp // 8) * (wp // 8), hp * wp
    m = T * p2 * 64 * 3 * 3 * 49                                               # stem
    m += 4 * T * p2 * 64 * 64 * 27                                             # layer1
    for p, ci, co in ((p4, 64, 128), (p8, 128, 256), (p8, 256, 512)):         # layer2..4
        m += T * p * co * ci * 27 + 3 * T * p * co * co * 27 + T * p * co * ci
    m += T * p8 * 256 * 512 * 27                                               # decoder 0
    m += T * p4 * 128 * 512 * 12 + T * p2 * 64 * 256 * 12                      # decoder 1, 2 (transposed: 3 x 2 x 2 taps)
    m += T * p2 * 64 * 128 * 27 + T * pp * 64 * 128 * 12                       # decoder 3, 4
    m += pp * 64 * 256 + pp * 3 * 64 * 49                                      # feature_fuse, outconv (3 outputs)
    return m


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
    for key, group in (("streamconv", "conv (streamconv)"), ("stem", "stem"), ("chan_sums", "gate sums"),
                       ("gate_kernel", "gate"), ("apply", "gate apply"), ("outconv", "outconv"),
                       ("frame_sums", "mean + pad"), ("prep", "mean + pad")):
        if key in name:
            return group
    return "other"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--h", type=int, default=1080)
    ap.add_argument("--w", type=int, default=1920)
    ap.add_argument("--windows", type=int, default=4, help="windows per library call (flavr_node.WINDOWS_PER_PASS)")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--torch-windows", type=int, default=4)
    ap.add_argument("--no-torch", action="store_true")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_flavr: no CUDA device")
    import __graft_entry__ as ge
    ge.load_package()
    from cfi_b200.engine import FlavrEngine

    sd = OV.synthetic_state_dict(0, "2x")
    eng = FlavrEngine(sd, device=0, dtype="float32")
    clip = O.synthetic_clip(a.frames, a.h, a.w, seed=7).cuda().contiguous()
    nwin = a.frames - 3
    out = torch.empty((nwin, a.h, a.w, 3), dtype=torch.float32, device="cuda")

    def step():
        for c0 in range(0, nwin, a.windows):
            c1 = min(nwin, c0 + a.windows)
            eng.forward(clip, list(range(c0, c1)), out=out[c0:c1])

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
    t = statistics.median(times)
    pl, pr, pt, pb = OV.pad_amounts(a.h, a.w)
    hp, wp = a.h + pt + pb, a.w + pl + pr
    macs = flavr_macs(hp, wp)
    res = dict(metric="flavr_2x_frames_per_s", value=round(nwin / t, 3), unit="interpolated frames/s",
               size=[a.h, a.w], padded=[hp, wp], frames=a.frames, windows_per_call=a.windows,
               step_s=[round(x, 4) for x in times], tflop_per_frame=round(2 * macs / 1e12, 3),
               tflops=round(2 * macs * nwin / t / 1e12, 1), out_finite=bool(torch.isfinite(out).all()),
               card=card(0))

    if not a.no_torch:
        torch.backends.cudnn.allow_tf32 = True  # PyTorch's default for convolutions, stated for the record
        sdc = {k: v.cuda() for k, v in sd.items()}
        nchw = clip.permute(0, 3, 1, 2)

        def torch_window(f):
            x = F.pad(nchw[f:f + 4], (pl, pr, pt, pb), mode="replicate")
            return OV.flavr_forward(sdc, x.unsqueeze(0))[0, :, pt:pt + a.h, pl:pl + a.w]

        with torch.no_grad():
            torch_window(0)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for f in range(a.torch_windows):
                y = torch_window(f)
            e1.record()
            torch.cuda.synchronize()
        tt = e0.elapsed_time(e1) / 1e3 / a.torch_windows
        diff = float((y.permute(1, 2, 0) - out[a.torch_windows - 1]).abs().max())
        res.update(torch_frames_per_s=round(1 / tt, 3), speedup_vs_torch=round(nwin / t * tt, 2),
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
    print(json.dumps(res), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
