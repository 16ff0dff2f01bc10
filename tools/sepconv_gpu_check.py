#!/usr/bin/env python
"""Sepconv on the GPU, checked against the unmodified reference's outputs (run on an H100;
tests/test_gpu_zsepconv.py runs it in a subprocess).

    python tools/sepconv_gpu_check.py

One JSON line per stage; exit code 0 only if every stage passed:
  forward_ref:<case> / forward:<case>   Network.forward through libvfi_b200.so with every conv on the CUDA-core checker /
                                        on the wgmma kernel vs tests/golden/sepconv_net_*.npz (PSNR >= 50 dB); the
                                        45x54 case has odd rows down the pyramid (crop-after-conv path of the decoder)
  batch                                 two pairs in one call == the two single calls
  node                                  SepconvVFI.vfi (multiplier 3) == the bisection of single engine calls
"""
import json
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from make_golden_sepconv import sepconv_cases, sepconv_inputs  # noqa: E402
from oracle import sepconv as OS  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
RESULTS = []


def report(stage, ok, **kw):
    row = dict(stage=stage, ok=bool(ok), **kw)
    RESULTS.append(row)
    print(json.dumps(row), flush=True)


def psnr(a, b):
    mse = float(((a.double() - b.double()) ** 2).mean())
    return 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)


def main():
    import __graft_entry__ as ge
    ge.load_package()
    from cfi_b200.engine import SepconvEngine
    import cfi_b200.sepconv_node as SN

    for use_ref, stage in ((True, "forward_ref"), (False, "forward")):
        for name, cfg in sorted(sepconv_cases().items()):
            try:
                ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"]).permute(0, 2, 3, 1)
                eng = SepconvEngine(OS.synthetic_state_dict(cfg["seed"]), device=0)
                eng.set_ref(use_ref)
                fr = sepconv_inputs(cfg).cuda().contiguous()
                out = eng.forward(fr, [0], [1])
                torch.cuda.synchronize()
                p = psnr(out.cpu(), ref)
                report(f"{stage}:{name}", p >= 50.0 and bool(torch.isfinite(out).all()), psnr_db=round(p, 2),
                       max_abs=float((out.cpu() - ref).abs().max()), launches=eng.launch_count())
                eng.close()
            except Exception as e:
                report(f"{stage}:{name}", False, error=repr(e)[:300])
    try:
        eng = SepconvEngine(OS.synthetic_state_dict(5), device=0)
        fr = sepconv_inputs(dict(kind="node", n=3, h=40, w=56, clip_seed=60)).cuda().contiguous()
        both = eng.forward(fr, [0, 1], [1, 2])
        one = torch.cat([eng.forward(fr, [0], [1]), eng.forward(fr, [1], [2])])
        report("batch", bool(torch.equal(both, one)), max_abs=float((both - one).abs().max()))
        (out,) = SN.SepconvVFI().vfi("sepconv.pth", fr.cpu(), multiplier=3, _engine=eng)
        x = fr.cpu().permute(0, 3, 1, 2)
        mid = eng.middle_frame(x[0:1], x[1:2]).cpu()
        # generic_frame_loop, multiplier 3 -> n = 2 in-between frames: bisection with the shared midpoint dropped
        left = eng.middle_frame(x[0:1], mid).cpu().permute(0, 2, 3, 1)[0]
        report("node", out.shape == (7, 40, 56, 3) and bool(torch.equal(out[1], left)) and bool(torch.equal(out[0], fr.cpu()[0])),
               shape=list(out.shape))
        # multiplier 2: the node's pipelined path (NHWC frames, staged uploads, downloads into the output's slots) must equal
        # the reference loop it replaces (frame_loop.generic_frame_loop), also with a skip list and an odd number of pairs
        from cfi_b200.frame_loop import generic_frame_loop
        from cfi_b200.node import InterpolationStateList
        fr6 = sepconv_inputs(dict(kind="node", n=6, h=40, w=56, clip_seed=61)).contiguous()
        for states in (None, InterpolationStateList([1, 3], True)):
            (fast,) = SN.SepconvVFI().vfi("sepconv.pth", fr6, multiplier=2, optional_interpolation_states=states, _engine=eng)
            slow = generic_frame_loop("SepconvVFI", fr6.permute(0, 3, 1, 2), 10, 2, lambda a, b, t, m: m.middle_frame(a, b), eng,
                                      interpolation_states=states, use_timestep=False, dtype=torch.float32).permute(0, 2, 3, 1)
            report("node_x2_pipelined" + ("" if states is None else "_skip"), fast.shape == slow.shape and bool(torch.equal(fast, slow)),
                   shape=list(fast.shape))
        eng.close()
    except Exception as e:
        report("batch/node", False, error=repr(e)[:300])

    bad = [r["stage"] for r in RESULTS if not r["ok"]]
    print(json.dumps(dict(summary=True, stages=len(RESULTS), failed=bad)), flush=True)
    out_path = os.environ.get("VFI_CHECK_JSONL")  # optional: every stage's record as one JSON line each
    if out_path:
        with open(out_path, "w") as fh:
            for r in RESULTS:
                fh.write(json.dumps(r) + "\n")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
