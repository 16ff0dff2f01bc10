#!/usr/bin/env python
"""One or more device-resident passes of the RIFE forward schedule and nothing else - the command ncu wraps for launch
lists and `--set full` captures (bench.py itself also runs the node, the CPU leg and the stand-alone kernel timings).

    ncu --metrics gpu__time_duration.sum --clock-control none -s <launches of the warm-up pass> -c 60 --csv \
        --log-file launches.csv python tools/profile_step.py --frames 9 --iters 2
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402
from oracle import rife46 as O  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=9, help="source frames: frames - 1 pairs = one pass of 8 by default")
    ap.add_argument("--iters", type=int, default=2)
    ap.add_argument("--arch", default="4.6")
    ap.add_argument("--dtype", default="float32")
    ap.add_argument("--h", type=int, default=1080)
    ap.add_argument("--w", type=int, default=1920)
    a = ap.parse_args()
    ge.load_package()
    from cfi_b200.engine import Rife46Engine
    eng = Rife46Engine(O.synthetic_state_dict(0, arch=a.arch), 0, a.dtype, batch=8, arch=a.arch)
    clip = O.synthetic_clip(a.frames, a.h, a.w, seed=1234).cuda()
    n = a.frames - 1
    out = torch.empty((n, a.h, a.w, 3), dtype=torch.float32, device="cuda")
    for _ in range(a.iters):
        eng.forward(clip, list(range(n)), list(range(1, n + 1)), [0.5] * n, out=out)
    torch.cuda.synchronize()
    print("launches", eng.launch_count())
    eng.close()


if __name__ == "__main__":
    main()
