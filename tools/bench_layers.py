#!/usr/bin/env python
"""Time every conv layer of the RIFE-4.6 path at the 1080p geometry (kernel only, CUDA events) and print
TFLOP/s per layer.  Usage: python tools/bench_layers.py [--batch 4] [--dtype float16] [--json out.json]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402
from oracle import rife46 as O  # noqa: E402

BLOCK_C = (192, 128, 96, 64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--dtype", default="float16")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--json", default="")
    ap.add_argument("--only", default="", help="block:layer, e.g. 3:2")
    ap.add_argument("--lib", default="", help="alternate libvfi_b200 build (diagnostic builds)")
    a = ap.parse_args()
    ge.load_package()
    if a.lib:
        from cfi_b200 import _lib
        _lib.LIB_PATH = os.path.abspath(a.lib)
    from cfi_b200.engine import Rife46Engine
    eng = Rife46Engine(O.synthetic_state_dict(0), 0, a.dtype)
    tdt = torch.float16 if a.dtype != "bfloat16" else torch.bfloat16
    Hp, Wp = 1088, 1920
    B = a.batch
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    rows = []
    for blk, s in enumerate((8, 4, 2, 1)):
        c = BLOCK_C[blk]
        Hs, Ws = Hp // s, Wp // s
        specs = [(0, (B, Hs // 2, Ws // 2, 64), (B, Hs // 4, Ws // 4, 2 * c)),
                 (1, (B, Hs // 4, Ws // 4, 2 * c), (B, Hs // 4, Ws // 4, c)),
                 (2, (B, Hs // 4, Ws // 4, c), (B, Hs // 4, Ws // 4, c)),
                 (10, (B, Hs // 4, Ws // 4, c), None)]
        for layer, ishape, oshape in specs:
            if a.only and a.only != f"{blk}:{layer}":
                continue
            x = (0.1 * torch.randn(ishape, device="cuda")).to(tdt)
            if layer == 10:
                out = torch.empty(B, Hs, Ws, 4, device="cuda")
                om = torch.empty(B, Hs, Ws, device="cuda")
            else:
                out = torch.empty(oshape, dtype=tdt, device="cuda")
                om = None
            pl = eng.layer_plan(blk, layer)
            for _ in range(3):
                eng.debug_layer(blk, layer, x, out, om)
            torch.cuda.synchronize()
            ts = []
            for _ in range(a.iters):
                flush.zero_()
                e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
                e0.record()
                eng.debug_layer(blk, layer, x, out, om)
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            ms = sorted(ts)[len(ts) // 2]
            cells = ishape[0] * ishape[1] * ishape[2]
            flops = 2.0 * pl["macs_per_cell"] * cells
            act_bytes = x.numel() * 2 + (out.numel() * out.element_size() + (om.numel() * 4 if om is not None else 0))
            row = dict(block=blk, layer=layer, c=c, grid=list(ishape[1:3]), batch=B, ms=ms, tflops=flops / ms / 1e9,
                       gbs=act_bytes / ms / 1e6, **pl)
            rows.append(row)
            print(json.dumps(row))
    if a.json:
        json.dump(rows, open(a.json, "w"), indent=1)
    eng.close()


if __name__ == "__main__":
    main()
