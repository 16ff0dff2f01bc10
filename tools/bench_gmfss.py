#!/usr/bin/env python
"""GMFSS Fortuna harness (BASELINE.json configs[3]: GMFSS Fortuna union, 2x, 720p on 1 x H100; `bench.py` metric family).

    python tools/bench_gmfss.py [--ckpt GMFSS_fortuna_union | GMFSS_fortuna] [--h 720 --w 1280] [--steps 3] [--warmup 2]

One step = one interpolated frame of a device-resident 720p pair through gmfss.GMFSS.interpolate (pad to 768 x 1280, GMFlow in
both directions, MetricNet, FeatureNet x 2, eight soft splats, RIFE 4.6 (union only), GridNet, crop).  `--ckpt` picks the
node's checkpoint: `GMFSS_fortuna_union` (default) or the base model `GMFSS_fortuna` (no RIFE, 12-channel GridNet input).
Prints ONE JSON line: frames/s, the split reuse / inference, fp32 MACs per frame counted from the calls, achieved TFLOP/s
against the fp32 FMA rate, the card's name and power limit, and the CPU oracle (oracle/gmfss.py for union, oracle/gmfss_base.py for base == the
reference's PyTorch-CPU path) on a small pair scaled by pixel count.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
FP32_FMA_TFLOPS = 67.0  # H100 SXM data sheet, FP32
VARIANT = {"GMFSS_fortuna_union": "union", "GMFSS_fortuna": "base"}


def card(index: int) -> dict:
    """name and power limit of the card the numbers come from (read only: nvidia-smi --query-gpu)"""
    import torch
    info = {"name": torch.cuda.get_device_name(index), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ckpt", choices=list(VARIANT), default="GMFSS_fortuna_union")
    ap.add_argument("--h", type=int, default=720)
    ap.add_argument("--w", type=int, default=1280)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    import __graft_entry__ as ge
    ge.load_package()
    from cfi_b200.gmfss import build_gpu_model
    from oracle import film as OF
    from oracle import gmfss as OG
    from oracle import gmfss_base as GB
    from oracle import gmfss_weights as GW
    variant = VARIANT[a.ckpt]
    W, O = (GW, OG) if variant == "union" else (GB, GB)   # seeded weights, CPU oracle
    sds = W.synthetic_state_dicts(0)
    m = build_gpu_model(sds, 0)
    # count the multiply-accumulates of the conv / gemm calls of one frame
    macs = {"n": 0}
    conv0, convt0, lin0, bmm0 = m.o.conv, m.o.convt4, m.o.linear, m.o.bmm

    def conv(x, w, *k, **kw):
        out = conv0(x, w, *k, **kw)
        macs["n"] += out.shape[0] * w.shape[0] * out.shape[2] * out.shape[3] * w.shape[1] * w.shape[2] * w.shape[3]
        return out

    def convt(x, w, *k, **kw):
        out = convt0(x, w, *k, **kw)
        macs["n"] += x.shape[0] * x.shape[2] * x.shape[3] * w.shape[0] * w.shape[1] * 16
        return out

    def lin(x, w, *k, **kw):
        macs["n"] += (x.numel() // x.shape[-1]) * w.shape[0] * w.shape[1]
        return lin0(x, w, *k, **kw)

    def bmm(a_, b_, bt, *k, **kw):
        macs["n"] += a_.shape[0] * a_.shape[1] * a_.shape[2] * (b_.shape[1] if bt else b_.shape[2])
        return bmm0(a_, b_, bt, *k, **kw)

    m.o.conv, m.o.convt4, m.o.linear, m.o.bmm = conv, convt, lin, bmm
    fr = OF.synthetic_clip(2, a.h, a.w, seed=1234).permute(0, 3, 1, 2).contiguous().cuda()
    f0, f1 = fr[0:1].contiguous(), fr[1:2].contiguous()
    out = None
    for _ in range(max(a.warmup, 1)):
        macs["n"] = 0
        out = m.interpolate(f0, f1, 0.5)
    torch.cuda.synchronize()
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    ms_reuse = ms_inf = 0.0
    ph, pw = ((a.h - 1) // 64 + 1) * 64, ((a.w - 1) // 64 + 1) * 64
    for _ in range(a.steps):
        macs["n"] = 0   # (per frame)
        i0, i1 = m.o.new(1, 3, ph, pw), m.o.new(1, 3, ph, pw)
        e[0].record()
        m.o.copy_slice(f0, i0, 3)
        m.o.copy_slice(f1, i1, 3)
        st = m.reuse(i0, i1)
        e[1].record()
        out = m.inference(st, 0.5)
        e[2].record()
        torch.cuda.synchronize()
        ms_reuse += e[0].elapsed_time(e[1])
        ms_inf += e[1].elapsed_time(e[2])
    ms = (ms_reuse + ms_inf) / a.steps
    tf = 2.0 * macs["n"] / (ms * 1e-3) / 1e12
    line = {"metric": f"interpolated frames/sec @{a.w}x{a.h} GMFSS Fortuna ({variant}) 2x", "value": 1e3 / ms, "unit": "frames/s", "n_gpus": 1,
            "steps": a.steps, "warmup": a.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32", "dtype_note": "gmops fp32 on CUDA cores" + ("; the RIFE 4.6 sub-model fp16 operands / fp32 accumulate"
                                                                         if variant == "union" else "; no RIFE sub-model"),
            "data": "synthetic", "gpu": card(0),
            "config": {"workload": f"GMFSS Fortuna {variant} ({a.ckpt}), 2x, one {a.h}x{a.w} pair per step, device resident"
                                   + (" (BASELINE configs[3])" if variant == "union" else ""),
                       "padded": [ph, pw],
                       "weights": f"seeded synthetic ({W.__name__}.synthetic_state_dicts(0)); no checkpoint ships"},
            "ms_reuse": ms_reuse / a.steps, "ms_inference": ms_inf / a.steps, "finite": bool(torch.isfinite(out).all()),
            "roofline": {"bound": "fp32 FMA", "kernel": "whole frame (gmops conv / gemm + element-wise + splats" + (" + RIFE)" if variant == "union" else ")"), "achieved": tf,
                         "peak": FP32_FMA_TFLOPS, "unit": "TFLOP/s", "frac": tf / FP32_FMA_TFLOPS, "gmacs_per_frame": macs["n"] / 1e9,
                         "peak_source": "H100 SXM data sheet (FP32)", "traffic": None}}
    if not a.no_cpu:
        torch.set_num_threads(min(32, os.cpu_count() or 1))
        hs, ws = 192, 256
        small = OF.synthetic_clip(2, hs, ws, seed=7).permute(0, 3, 1, 2).contiguous()
        t0 = time.perf_counter()
        with torch.no_grad():
            O.interpolate(sds, small[0:1], small[1:2], 0.5)
        sec = time.perf_counter() - t0
        line["cpu_baseline"] = {"value": 1.0 / (sec * (ph * pw) / (hs * ws)), "unit": "frames/s", "cores": torch.get_num_threads(), "kind": "port",
                                "sample": f"one {hs}x{ws} pair ({sec:.1f} s) scaled by pixel count to the padded {ph}x{pw}; {O.__file__[len(ROOT) + 1:]} == "
                                          "the reference's PyTorch-CPU path with its splat restated on the CPU"}
    print(json.dumps(line))
    if m._engine is not None:
        m._engine.close()


if __name__ == "__main__":
    main()
