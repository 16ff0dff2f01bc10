#!/usr/bin/env python
"""Time the `vfi_models.ops` replacement kernels (kernel only, CUDA events, L2 flushed between launches) at the shapes
SURVEY.md section 8 (a11, a12) names and print the achieved algorithmic GB/s / GFLOP/s next to the measured peaks.

    python tools/bench_ops.py [--json out.json] [--small]

  warp       : rife_arch.warp, NHWC fp32 [8,1088,1920,4]                      bytes = (C + 2 + C) * 4 per pixel
  softsplat  : GMFSS shapes @768x1280 (flows at 384x640): [1,64,384,640], [1,129,192,320], [1,193,96,160], sum mode
               bytes = read C + 2, memset + write C (x4 B); atomics = 4 per element
  costvol/corr: 9x9 volumes on [1,64,96,160] and [1,128,192,320]             flop = 2 * 81 * C per pixel
  sepconv    : K = 51 on a 4-channel frame (config 5 is 3840x2160; --small: 1920x1080)   flop = 2 * 51*51 * 4 per pixel
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402


def timed(fn, flush, iters=8, warm=2):
    ts = []
    for i in range(warm + iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        if i >= warm:
            ts.append(a.elapsed_time(b))
    return sum(ts) / len(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default="")
    ap.add_argument("--small", action="store_true")
    a = ap.parse_args()
    ge.load_package()
    import cfi_b200.ops as OPS
    from cfi_b200.engine import Rife46Engine
    from oracle import rife46 as O
    peaks = {"hbm_gbs": 6585.1}
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        peaks = json.load(open(p))
    fp32_peak = 132 * 128 * 2 * 1.98e9 / 1e9  # GFLOP/s, H100 SXM CUDA-core FMA peak at the maximum SM clock
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    rows = []

    def add(name, shape, ms, bytes_, flops, note=""):
        r = dict(op=name, shape=shape, ms=ms, gbs=bytes_ / ms / 1e6, gflops=flops / ms / 1e6,
                 frac_hbm=bytes_ / ms / 1e6 / peaks["hbm_gbs"], frac_fp32=flops / ms / 1e6 / fp32_peak, note=note)
        rows.append(r)
        print(f"{name:10s} {str(shape):28s} {ms * 1e3:9.1f} us  {r['gbs']:8.1f} GB/s ({100 * r['frac_hbm']:5.1f}% HBM)  "
              f"{r['gflops']:9.1f} GFLOP/s ({100 * r['frac_fp32']:5.1f}% fp32)  {note}", flush=True)

    g = torch.Generator(device="cuda").manual_seed(0)
    # warp primitive
    eng = Rife46Engine(O.synthetic_state_dict(0), 0, "float32")
    img = torch.rand(8, 1088, 1920, 4, device="cuda", generator=g)
    fl = torch.nn.functional.interpolate(4 * torch.randn(8, 2, 34, 60, device="cuda", generator=g), size=(1088, 1920),
                                         mode="bilinear").permute(0, 2, 3, 1).contiguous()
    ms = timed(lambda: eng.warp(img, fl), flush)
    add("warp", (8, 1088, 1920, 4), ms, img.numel() * 4 * 2 + fl.numel() * 4, 0, "smooth +-4 px flow")
    del img, fl
    eng.close()
    # softsplat (sum)
    for c, h, w in ((64, 384, 640), (129, 192, 320), (193, 96, 160)):
        x = torch.randn(1, c, h, w, device="cuda", generator=g)
        f = torch.nn.functional.interpolate(6 * torch.randn(1, 2, h // 16, w // 16, device="cuda", generator=g),
                                            size=(h, w), mode="bilinear")
        ms = timed(lambda: OPS.softsplat_func.apply(x, f), flush)
        add("softsplat", (1, c, h, w), ms, (x.numel() * 3 + f.numel()) * 4, 8.0 * x.numel(),
            "sum mode; 4 atomics per element; bytes = read + memset + write")
        # soft mode (what GMFSS calls): the reference's cat -> splat -> slice -> divide chain vs the fused two-launch form
        m = torch.randn(1, 1, h, w, device="cuda", generator=g)
        soft_bytes = (x.numel() * 4 + f.numel() + 3 * m.numel()) * 4      # read C + 3, memset C + 1, splat, normalise r/w C
        ms = timed(lambda: OPS.softsplat(x, f, m, "soft"), flush)
        add("softsplat_soft", (1, c, h, w), ms, soft_bytes, 8.0 * x.numel(), "vfi_softsplat_weighted, two launches")
    # 9x9 volumes
    for c, h, w in ((64, 96, 160), (128, 192, 320)):
        one = torch.randn(1, c, h, w, device="cuda", generator=g)
        two = torch.randn(1, c, h, w, device="cuda", generator=g)
        by = (2 * c + 81) * h * w * 4
        ms = timed(lambda: OPS.costvol_func.apply(one, two), flush)
        add("costvol", (1, c, h, w), ms, by, 2.0 * 81 * c * h * w)
        ms = timed(lambda: OPS.FunctionCorrelation(one, two), flush)
        add("corr", (1, c, h, w), ms, by, 2.0 * 81 * c * h * w)
    # sepconv K = 51, RGB + ones
    h, w = (1080, 1920) if a.small else (2160, 3840)
    x = torch.rand(1, 4, h + 50, w + 50, device="cuda", generator=g)
    ver = torch.randn(1, 51, h, w, device="cuda", generator=g) / 51
    hor = torch.randn(1, 51, h, w, device="cuda", generator=g) / 51
    ms = timed(lambda: OPS.sepconv_func.apply(x, ver, hor), flush, iters=4, warm=1)
    add("sepconv", (1, 4, h, w, "K=51"), ms, (x.numel() + ver.numel() * 2 + 4 * h * w) * 4, 2.0 * 51 * 51 * 4 * h * w,
        f"VFI_SEPCONV_PY={os.environ.get('VFI_SEPCONV_PY', '2 (default)')}")
    if a.json:
        json.dump(rows, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
