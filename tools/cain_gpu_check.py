#!/usr/bin/env python
"""CAIN on the GPU, checked stage by stage (run on an H100; tests/test_gpu_zcain.py runs it in a subprocess).

    python tools/cain_gpu_check.py [--parent-src DIR]

Stages, each reported as one JSON line {"stage": ..., "ok": ..., ...}; exit code 0 only if every stage passed:
  elem:<dtype>:<kernel>  the element-wise kernels through vfi_cain_debug_elem on a 130 x 135 frame (a 32 x 32 trunk grid,
                         34 x 34 bordered) against torch: prep (mean, F.pad(mode="reflect") to 256 x 256, space-to-depth,
                         zero border), the reflected border (F.pad(mode="reflect") by one cell, bit-exact), the zero
                         border with a sum (bit-exact), channel attention (mean, 192 -> 12 -> 192 gate, x * gate + res,
                         the border from the mirrored cells; NaN in the inputs' borders must not reach the output), and
                         final (depth-to-space, crop, + mean); fp16 and bf16
  forward_ref / forward  the model goldens through libvfi_b200.so on the checker / on the wgmma kernel vs the unmodified
                         reference's output (tests/golden/cain_*.npz): PSNR >= 50 dB
  node                   CAIN_VFI.vfi vs the unmodified reference node (tests/golden/cain_node_*.npz): interpolated
                         frames PSNR >= 50 dB, pass-through frames bit-exact
  refuse                 a frame ReflectionPad2d cannot pad is refused before any launch
  parent:<model>         with --parent-src (a checkout of the parent commit): FILM, Sepconv, FLAVR and IFRNet outputs on
                         seeded inputs bit-identical between this library and the parent's, built in a temp directory
The oracle / goldens are the checker here, never the thing measured.
"""
import json
import math
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from make_golden_cain import cain_cases, cain_inputs, case_state_dict  # noqa: E402
from oracle import cain as OC  # noqa: E402
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


def rel(a, b):
    return float((a.float() - b.float()).abs().max()) / (float(b.float().abs().max()) + 1e-12)


def elem_stages(dt, sd):
    """The five element-wise kernels of one operand type on a 130 x 135 frame."""
    from cfi_b200.engine import CainEngine
    td = torch.float16 if dt == "float32" else torch.bfloat16
    tol = 2e-3 if dt == "float32" else 1.6e-2
    eng = CainEngine(sd, device=0, dtype=dt)
    H, W = 130, 135
    geo = OC.geometry(H, W)
    h, w, t, l = geo["gh"], geo["gw"], geo["top"], geo["left"]
    g = torch.Generator().manual_seed(3)
    img = torch.rand(2, 1, 3, H, W, generator=g).cuda()
    nan = float("nan")

    def bordered(c=192, fill=nan):
        x = torch.full((h + 2, w + 2, c), fill, dtype=td)
        x[1:-1, 1:-1] = (torch.rand(h, w, c, generator=g) * 2 - 1).to(td)
        return x.cuda()

    def interior(x):
        return x[1:-1, 1:-1].float().permute(2, 0, 1)[None]

    def reflect1(y):   # [1, C, h, w] -> bordered [h + 2, w + 2, C]
        return F.pad(y, (1, 1, 1, 1), mode="reflect")[0].permute(1, 2, 0)

    # prep
    out = torch.full((h + 2, w + 2, 384), nan, dtype=td, device="cuda")
    eng.debug_elem(0, H, W, img0=img[0], img1=img[1], out=out)
    ref = torch.zeros(h + 2, w + 2, 384, device="cuda")
    pads = (l, geo["wp"] - W - l, t, geo["hp"] - H - t)
    for f in range(2):
        x = F.pad(img[f] - img[f].mean(dim=(2, 3), keepdim=True), pads, mode="reflect")
        ref[1:-1, 1:-1, 192 * f:192 * (f + 1)] = OC.space_to_depth(x)[0].permute(1, 2, 0)
    border = torch.ones(h + 2, w + 2, dtype=torch.bool)
    border[1:-1, 1:-1] = False
    e = rel(out, ref.to(td))
    report(f"elem:{dt}:prep", e <= tol and bool((out[border.cuda()] == 0).all()), rel_err=e)

    # reflected border: a copy, bit-exact
    x = bordered()
    want = reflect1(interior(x)).to(td)
    eng.debug_elem(1, H, W, out=x)
    torch.cuda.synchronize()
    report(f"elem:{dt}:border_reflect", torch.equal(x.view(torch.int16), want.view(torch.int16)))

    # zero border + sum: one rounding, as torch does it
    x, a = bordered(), bordered()
    want = torch.zeros_like(x)
    want[1:-1, 1:-1] = (x[1:-1, 1:-1].float() + a[1:-1, 1:-1].float()).to(td)
    eng.debug_elem(2, H, W, res=a, out=x)
    torch.cuda.synchronize()
    report(f"elem:{dt}:border_zero_add", torch.equal(x.view(torch.int16), want.view(torch.int16)))

    # channel attention of RCAB 37 (group 3, block 1); NaN borders on both inputs
    k = 37
    p = f"{OC.PREFIX}body.{k // 12}.body.{k % 12}.body.3.conv_du."
    x, r = bordered(), bordered()
    out = torch.full_like(x, nan)
    eng.debug_elem(3, H, W, x=x, res=r, out=out, rcab=k)
    xi, ri = interior(x).double(), interior(r).double()
    m = xi.mean(dim=(2, 3), keepdim=True)
    wd = {n: sd[p + n].double().cuda() for n in ("0.weight", "0.bias", "2.weight", "2.bias")}
    gate = torch.sigmoid(F.conv2d(F.relu(F.conv2d(m, wd["0.weight"], wd["0.bias"])), wd["2.weight"], wd["2.bias"]))
    want = reflect1(xi * gate + ri)
    e = rel(out, want)
    report(f"elem:{dt}:attention", e <= tol and not torch.isnan(out).any(), rel_err=e,
           gate_range=[round(float(gate.min()), 4), round(float(gate.max()), 4)])

    # final
    x = bordered()
    out = torch.full((1, 3, H, W), nan, device="cuda")
    eng.debug_elem(4, H, W, img0=img[0], img1=img[1], x=x, out=out)
    y = OC.depth_to_space(interior(x))[:, :, t:t + H, l:l + W]
    want = y + (img[0].mean(dim=(2, 3), keepdim=True) + img[1].mean(dim=(2, 3), keepdim=True)) / 2
    e = float((out - want).abs().max())
    report(f"elem:{dt}:final", e <= 1e-5, max_abs=e)
    eng.close()


def parent_outputs(path):
    """FILM, Sepconv, FLAVR and IFRNet on seeded inputs with this process's library -> npz (the parent comparison)."""
    import __graft_entry__ as ge
    ge.load_package()
    from cfi_b200.engine import FilmEngine, FlavrEngine, IfrnetEngine, SepconvEngine
    from oracle import flavr as OV
    from oracle import ifrnet as OI
    from oracle import sepconv as OS
    fr = OF.synthetic_clip(5, 72, 104, seed=61).cuda()
    film = FilmEngine(OF.synthetic_state_dict(1, 2.0), device=0, dtype="float32").forward(fr, [0, 1], [1, 2]).cpu().numpy()
    sep = SepconvEngine(OS.synthetic_state_dict(5), device=0).forward(fr, [0, 1], [1, 2]).cpu().numpy()
    flavr = FlavrEngine(OV.synthetic_state_dict(0, "4x"), device=0).forward(fr.contiguous(), [0, 1]).cpu().numpy()
    x = fr.permute(0, 3, 1, 2).contiguous()
    ifr = IfrnetEngine(OI.synthetic_state_dict("L", 0), device=0).forward(x[0:1], x[1:2], 0.5, 1.0).cpu().numpy()
    np.savez(path, film=film, sep=sep, flavr=flavr, ifrnet=ifr)


def parent_stage(parent_src):
    with tempfile.TemporaryDirectory() as td:
        src = os.path.join(td, "parent")
        shutil.copytree(parent_src, src, ignore=shutil.ignore_patterns("*.so", "__pycache__"))
        r = subprocess.run([sys.executable, "-c", "import __graft_entry__ as g; g.build()"], cwd=src, capture_output=True,
                           text=True)
        if r.returncode != 0:
            report("parent:build", False, error=r.stderr[-2000:])
            return
        outs = []
        for root in (ROOT, src):
            p = os.path.join(td, f"out{len(outs)}.npz")
            r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "cain_gpu_check.py"), "--parent-outputs", p],
                               cwd=root, capture_output=True, text=True, env=dict(os.environ, VFI_CHECK_ROOT=root))
            if r.returncode != 0:
                report("parent:run", False, root=root, error=r.stderr[-2000:])
                return
            outs.append(np.load(p))
        for key in ("film", "sep", "flavr", "ifrnet"):
            a, b = outs[0][key], outs[1][key]
            report(f"parent:{key}", a.shape == b.shape and a.tobytes() == b.tobytes(), shape=list(a.shape),
                   max_abs_diff=float(np.abs(a - b).max()))


def main():
    if "--parent-outputs" in sys.argv:
        root = os.environ.get("VFI_CHECK_ROOT", ROOT)
        sys.path.insert(0, root)
        parent_outputs(sys.argv[sys.argv.index("--parent-outputs") + 1])
        return 0
    import __graft_entry__ as ge
    ge.load_package()
    from cfi_b200._lib import VfiError
    from cfi_b200.engine import CainEngine
    import cfi_b200.cain_node as CN

    sd = OC.synthetic_state_dict(0)
    for dt in ("float32", "bfloat16"):
        try:
            elem_stages(dt, sd)
        except Exception as e:  # keep going: later stages still tell something
            report(f"elem:{dt}", False, error=repr(e)[:300])

    for use_ref, stage in ((True, "forward_ref"), (False, "forward")):
        for name, cfg in sorted(cain_cases().items()):
            if cfg["kind"] != "net":
                continue
            try:
                ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
                e2 = CainEngine(case_state_dict(cfg), device=0, dtype="float32")
                e2.set_ref(use_ref)
                x = cain_inputs(cfg)[..., :3].permute(0, 3, 1, 2).contiguous().cuda()
                out = e2.forward(x[0:1].contiguous(), x[1:2].contiguous())
                torch.cuda.synchronize()
                p = psnr(out.cpu(), ref)
                report(f"{stage}:{name}", p >= 50.0, psnr_db=round(p, 2), max_abs=float((out.cpu() - ref).abs().max()),
                       launches=e2.launch_count())
                e2.close()
            except Exception as e:
                report(f"{stage}:{name}", False, error=repr(e)[:300])

    for name, cfg in sorted(cain_cases().items()):
        if cfg["kind"] != "node":
            continue
        try:
            ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
            e3 = CainEngine(case_state_dict(cfg), device=0, dtype="float32")
            fr = cain_inputs(cfg)
            st = None if cfg["states"] is None else CN.InterpolationStateList(list(cfg["states"][0]), cfg["states"][1])
            (out,) = CN.CAIN_VFI().vfi("pretrained_cain.pth", fr, multiplier=cfg["multiplier"],
                                       optional_interpolation_states=st, _engine=e3)
            src = fr[..., :3]
            passthru = [i for i in range(ref.shape[0]) if any(torch.equal(ref[i], s) for s in src)]
            mids = [i for i in range(ref.shape[0]) if i not in passthru]
            exact = out.shape == ref.shape and all(torch.equal(out[i], ref[i]) for i in passthru)
            p = psnr(out[mids], ref[mids]) if mids and out.shape == ref.shape else 0.0
            report(f"node:{name}", exact and p >= 50.0, psnr_db=round(p, 2), shape=list(out.shape),
                   passthrough=len(passthru), interpolated=len(mids))
            e3.close()
        except Exception as e:
            report(f"node:{name}", False, error=repr(e)[:300])

    try:
        e4 = CainEngine(sd, device=0)
        x = torch.rand(1, 3, 64, 40, device="cuda")
        out = torch.full_like(x, 7.0)
        n0 = e4.launch_count()
        try:
            e4.forward(x, x, out=out)
            refused, msg = False, ""
        except VfiError as err:
            refused, msg = True, str(err)
        torch.cuda.synchronize()
        report("refuse:64x40", refused and "cannot be reflection-padded" in msg and e4.launch_count() == n0
               and bool((out == 7.0).all()), message=msg[:200])
        e4.close()
    except Exception as e:
        report("refuse:64x40", False, error=repr(e)[:300])

    if "--parent-src" in sys.argv:
        try:
            parent_stage(sys.argv[sys.argv.index("--parent-src") + 1])
        except Exception as e:
            report("parent", False, error=repr(e)[:300])

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
