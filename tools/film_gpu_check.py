#!/usr/bin/env python
"""FILM on the GPU, checked stage by stage (run on an H100; tests/test_gpu_zfilm.py runs it in a subprocess).

    python tools/film_gpu_check.py [--quick]

Stages, each reported as one JSON line {"stage": ..., "ok": ..., ...}; exit code 0 only if every stage passed:
  conv:<group>.<layer>   one streamconv layer on random 16-bit inputs: wgmma kernel vs the CUDA-core checker (same
                         packed weights) and, for layers whose input channels are in reference order, vs torch conv2d
                         on the CPU with the layer's real weights
  forward_ref / forward  Interpolator.forward through libvfi_b200.so with every conv on the CUDA-core checker / on the
                         wgmma kernel, vs the unmodified reference's output (tests/golden/film_net_*.npz): PSNR >= 50 dB
                         on the frame only (the flows of every level, per pixel, and bf16 operands are checked by
                         tests/test_gpu_zfilm16.py)
  node                   FILM_VFI.vfi vs the unmodified reference node's output (tests/golden/film_node_*.npz)
The oracle / goldens are the checker here, never the thing measured.
"""
import json
import math
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from make_golden_film import film_cases, film_inputs  # noqa: E402
from oracle import film as OF  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
RESULTS = []


def report(stage, ok, **kw):
    row = dict(stage=stage, ok=bool(ok), **kw)
    RESULTS.append(row)
    print(json.dumps(row), flush=True)


def psnr(a, b):
    mse = float(((a.double() - b.double()) ** 2).mean())
    return 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)


def conv_stage(eng, sd, group, layer, name, ksize, act, B=2, H=37, W=29):
    """name: state_dict prefix when the layer's input channels are in reference order (else None)."""
    plan = eng.layer_plan(group, layer)
    c0, c1, n = plan["c0"], plan["c1"], plan["n_total"]
    g = torch.Generator().manual_seed(100 * group + layer)
    x0 = (torch.rand(B, H, W, c0, generator=g) - 0.5).half().cuda()
    x1 = (torch.rand(B, H, W, c1, generator=g) - 0.5).half().cuda() if c1 else None
    outs = []
    for impl in (1, 0):
        out = torch.full((B, H, W, n), float("nan"), dtype=torch.float16, device="cuda")
        eng.debug_conv(group, layer, x0, x1, out, B, H, W, impl=impl)
        torch.cuda.synchronize()
        outs.append(out.float().cpu())
    ref_k, tc = outs
    scale = float(ref_k.abs().max()) + 1e-6
    err_tc = float((tc - ref_k).abs().max()) / scale
    info = dict(plan=plan, rel_err_tc_vs_checker=err_tc, nan_tc=int(torch.isnan(tc).sum()), nan_ref=int(torch.isnan(ref_k).sum()))
    ok = err_tc <= 4e-3 and info["nan_tc"] == 0 and info["nan_ref"] == 0
    if name is not None:
        w = sd[name + ".weight"].half().float()
        b = sd[name + ".bias"]
        cin = w.shape[1]
        x = torch.cat([x0] + ([x1] if c1 else []), -1).float().cpu()[..., :cin].permute(0, 3, 1, 2)
        y = F.conv2d(x, w, b, padding="same")
        if act:
            y = F.leaky_relu(y, 0.2)
        y = y.permute(0, 2, 3, 1)
        err_t = float((ref_k[..., :y.shape[-1]] - y).abs().max()) / (float(y.abs().max()) + 1e-6)
        info["rel_err_checker_vs_torch"] = err_t
        ok = ok and err_t <= 4e-3
    report(f"conv:{group}.{layer}", ok, **info)


def main():
    quick = "--quick" in sys.argv
    import __graft_entry__ as ge
    ge.load_package()
    from cfi_b200.engine import FilmEngine
    import cfi_b200.film_node as FN

    sd = OF.synthetic_state_dict(0, 1.0)
    eng = FilmEngine(sd, device=0, dtype="float32")
    # ---- single layers: identity-mapped ones (checked against torch), then the remapped / two-tensor ones
    convs = [
        (0, 2, "extract.extract_sublevels.convs.1.0.0", 3, 1),    # 64 -> 128
        (0, 3, "extract.extract_sublevels.convs.1.1.0", 3, 1),    # 128 -> 128
        (0, 7, "extract.extract_sublevels.convs.3.1.0", 3, 1),    # 512 -> 512, 4 output splits
        (1, 4, "predict_flow._predictors.1._convs.0.0", 3, 1),    # level 1: cat(192, 192) -> 64, two tensors
        (1, 13, "predict_flow._predictor._convs.1.0", 3, 1),      # 256 -> 256
        (1, 15, "predict_flow._predictor._convs.3.0", 1, 1),      # 1x1 256 -> 128
        (1, 1, None, 3, 1),                                      # level 0: 32 (padded 64) -> 32 (padded 64)
        (1, 3, None, 1, 1),                                      # level 0: 1x1 -> 16 columns
        (2, 9, None, 2, 0),                                      # 2x2, no activation, 128 -> 64
        (2, 10, None, 3, 1),                                     # cat(aligned 192, 64) -> 64, remapped channels
        (2, 11, "fuse.convs.3.2.0", 3, 1),                         # 64 -> 64
    ]
    if not quick:
        convs += [(2, 0, None, 2, 0), (2, 1, None, 3, 1)]        # 1984 -> 512 (2x2), cat(1984, 512) -> 512
    for gl in convs:
        try:
            conv_stage(eng, sd, *gl)
        except Exception as e:  # keep going: later stages still tell something
            report(f"conv:{gl[0]}.{gl[1]}", False, error=repr(e)[:300])

    # ---- whole network vs the unmodified reference's outputs
    for use_ref, stage in ((True, "forward_ref"), (False, "forward")):
        for name, cfg in sorted(film_cases().items()):
            if cfg["kind"] != "net" or (quick and name != "film_net_72x104"):
                continue
            try:
                gold = np.load(os.path.join(GOLD, name + ".npz"))
                e2 = FilmEngine(OF.synthetic_state_dict(cfg["seed"], cfg["flow_gain"]), device=0, dtype="float32")
                e2.set_ref(use_ref)
                fr = film_inputs(cfg).cuda().contiguous()
                out = e2.forward(fr, [0], [1], clamp=False)
                torch.cuda.synchronize()
                ref = torch.from_numpy(gold["out"]).permute(0, 2, 3, 1)
                p = psnr(out.cpu(), ref)
                report(f"{stage}:{name}", p >= 50.0, psnr_db=round(p, 2), launches=e2.launch_count(),
                       gmacs=round(e2.last_macs() / 1e9, 2))
                e2.close()
            except Exception as e:
                report(f"{stage}:{name}", False, error=repr(e)[:300])

    # ---- node vs the unmodified reference node
    for name, cfg in sorted(film_cases().items()):
        if cfg["kind"] != "node" or (quick and name != "film_node_mlist"):
            continue
        try:
            ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
            e3 = FilmEngine(OF.synthetic_state_dict(cfg["seed"], cfg["flow_gain"]), device=0, dtype="float32")
            st = None if cfg["states"] is None else FN.InterpolationStateList(list(cfg["states"][0]), cfg["states"][1])
            (out,) = FN.FILM_VFI().vfi("film_net_fp32.pt", film_inputs(cfg), multiplier=cfg["multiplier"],
                                       optional_interpolation_states=st, _engine=e3)
            p = psnr(out, ref)
            report(f"node:{name}", out.shape == ref.shape and p >= 50.0, psnr_db=round(p, 2), shape=list(out.shape))
            e3.close()
        except Exception as e:
            report(f"node:{name}", False, error=repr(e)[:300])

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
