#!/usr/bin/env python
"""IFUnet on the GPU, checked stage by stage (run on an H100; tests/test_gpu_zifunet.py runs it in a subprocess).

    python tools/ifunet_gpu_check.py [--parent-src DIR]

Stages, each reported as one JSON line {"stage": ..., "ok": ..., ...}; exit code 0 only if every stage passed:
  elem:<dtype>:<kernel>  the element-wise kernels through vfi_ifunet_debug_elem against torch in fp32: the level-0 input
                         (resize at scale 1.5, the 7 -> 17 conv0 + PReLU, both ensemble images, the space-to-depth copy),
                         CBAM (channel gate from both pools, spatial gate with BatchNorm), the convex upsampling
                         (softmax over the 9 taps of unfold(L * flow)) and the frame warps (grid_sample, border,
                         align_corners=True); fp16 and bf16
  forward_ref / forward  the model goldens through libvfi_b200.so on the checker / on the wgmma kernel vs the unmodified
                         reference's output (tests/golden/ifunet_*.npz): PSNR >= 50 dB, each figure recorded
  node                   IFUnet_VFI.vfi vs the unmodified reference node (tests/golden/ifunet_node_*.npz): interpolated
                         frames PSNR >= 50 dB, pass-through frames bit-exact
  refuse                 scale_factor 0.25, 0.7 and 1.2 (where the reference raises) are refused before any launch
  parent:<model>         with --parent-src (a checkout of the parent commit): RIFE, FILM, Sepconv, FLAVR, IFRNet and
                         CAIN outputs on seeded inputs bit-identical between this library and the parent's, built in a
                         temp directory
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

from make_golden_ifunet import case_state_dict, ifunet_cases, ifunet_inputs  # noqa: E402
from oracle import film as OF  # noqa: E402
from oracle import ifunet as OU  # noqa: E402

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
    from cfi_b200.engine import IfunetEngine
    td = torch.float16 if dt == "float32" else torch.bfloat16
    tol = 2e-3 if dt == "float32" else 1.6e-2
    eng = IfunetEngine(sd, device=0, dtype=dt)
    sdc = {k: v.cuda() for k, v in sd.items()}
    g = torch.Generator().manual_seed(7)

    # level-0 input at scale 1.5, both ensemble images: cat(a, b, t) resized, conv0 + PReLU, space-to-depth
    H, W, s, t = 100, 150, 1.5, 1 / 3
    geo = OU.geometry(H, W, s)
    h0, w0 = geo["levels"][0]
    img = torch.rand(2, 1, 3, H, W, generator=g).cuda()
    out = torch.full((2, (h0 + 1) // 2, (w0 + 1) // 2, 128), float("nan"), dtype=td, device="cuda")
    eng.debug_elem(0, H, W, img0=img[0], img1=img[1], out=out, index=2, timestep=t, scale=s)
    p = (0, geo["wp"] - W, 0, geo["hp"] - H)
    i0, i1 = F.pad(img[0], p), F.pad(img[1], p)
    tp = torch.ones_like(i0[:, :1]) * t
    want = torch.zeros_like(out, dtype=torch.float32)
    for b, x in enumerate((torch.cat((i0, i1, tp), 1), torch.cat((i1, i0, 1 - tp), 1))):
        x = OU.resize(x, s)
        y = F.prelu(F.conv2d(x, sdc["flownet.fmap.conv0.0.weight"], sdc["flownet.fmap.conv0.0.bias"]),
                    sdc["flownet.fmap.conv0.1.weight"])
        y = F.pad(y, (0, w0 % 2, 0, h0 % 2))[0]
        for q in range(4):
            want[b, :, :, q * 24:q * 24 + 17] = y[:, q >> 1::2, q & 1::2].permute(1, 2, 0)
    e = rel(out, want)
    report(f"elem:{dt}:flow_in", e <= tol and not torch.isnan(out).any(), rel_err=e)

    # CBAM of FeatureNet conv3 (128 channels) in place
    h, w, C = 34, 60, 128
    x = (torch.rand(1, h, w, C, generator=g) * 2 - 1).to(td).cuda()
    xin = x.float().permute(0, 3, 1, 2).double()
    eng.debug_elem(1, h, w, out=x, index=1)
    sdd = {k: v.double() for k, v in sdc.items() if v.is_floating_point()}
    want = OU._cbam(sdd, "flownet.fmap.conv3.cbam.", xin, {})
    e = rel(x.float().permute(0, 3, 1, 2), want)
    report(f"elem:{dt}:cbam", e <= tol, rel_err=e)

    # convex upsampling of IFBlock 1 (L = 8)
    L, h, w = 8, 9, 13
    fl = (torch.randn(1, h, w, 4, generator=g) * 3).cuda()
    mk = (torch.randn(1, h, w, 9 * L * L, generator=g) * 2).to(td).cuda()
    up = torch.full((1, L * h, L * w, 4), float("nan"), device="cuda")
    eng.debug_elem(2, h, w, x=fl, y=mk, out=up, index=1)
    m = torch.softmax(mk.float().permute(0, 3, 1, 2).reshape(1, 1, 9, L, L, h, w), dim=2)
    uf = F.unfold(L * fl.permute(0, 3, 1, 2), [3, 3], padding=1).view(1, 4, 9, 1, 1, h, w)
    want = torch.sum(m * uf, dim=2).permute(0, 1, 4, 2, 5, 3).reshape(1, 4, L * h, L * w).permute(0, 2, 3, 1)
    e = float((up - want).abs().max())
    report(f"elem:{dt}:convex", e <= 1e-4, max_abs=e)

    # warps of a pair
    H, W = 100, 150
    Hp, Wp = 128, 192
    flow = (torch.randn(Hp, Wp, 4, generator=g) * 6).cuda()
    wout = torch.full((2, 3, Hp, Wp), float("nan"), device="cuda")
    eng.debug_elem(3, H, W, img0=img[0], img1=img[1], x=flow, out=wout)
    fnchw = flow.permute(2, 0, 1)[None]
    want = torch.cat([OU.warp(F.pad(img[0], (0, Wp - W, 0, Hp - H)), fnchw[:, :2]),
                      OU.warp(F.pad(img[1], (0, Wp - W, 0, Hp - H)), fnchw[:, 2:4])], 0)
    e = float((wout - want).abs().max())
    report(f"elem:{dt}:warp", e <= 1e-4, max_abs=e)
    eng.close()


def parent_outputs(path):
    """RIFE, FILM, Sepconv, FLAVR, IFRNet and CAIN on seeded inputs with this process's library -> npz."""
    import __graft_entry__ as ge
    ge.load_package()
    from cfi_b200.engine import CainEngine, FilmEngine, FlavrEngine, IfrnetEngine, Rife46Engine, SepconvEngine
    from oracle import cain as OC
    from oracle import flavr as OV
    from oracle import ifrnet as OI
    from oracle import rife46 as OR
    from oracle import sepconv as OS
    fr = OF.synthetic_clip(5, 72, 104, seed=61).cuda()
    rife = Rife46Engine(OR.synthetic_state_dict(0), 0, "float32").forward(fr, [0, 1], [1, 2], [0.5, 0.5]).cpu().numpy()
    film = FilmEngine(OF.synthetic_state_dict(1, 2.0), device=0, dtype="float32").forward(fr, [0, 1], [1, 2]).cpu().numpy()
    sep = SepconvEngine(OS.synthetic_state_dict(5), device=0).forward(fr, [0, 1], [1, 2]).cpu().numpy()
    flavr = FlavrEngine(OV.synthetic_state_dict(0, "4x"), device=0).forward(fr.contiguous(), [0, 1]).cpu().numpy()
    x = fr.permute(0, 3, 1, 2).contiguous()
    ifr = IfrnetEngine(OI.synthetic_state_dict("L", 0), device=0).forward(x[0:1], x[1:2], 0.5, 1.0).cpu().numpy()
    cain = CainEngine(OC.synthetic_state_dict(0), device=0).forward(x[0:1].contiguous(), x[1:2].contiguous()).cpu().numpy()
    np.savez(path, rife=rife, film=film, sep=sep, flavr=flavr, ifrnet=ifr, cain=cain)


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
            r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "ifunet_gpu_check.py"), "--parent-outputs", p],
                               cwd=root, capture_output=True, text=True, env=dict(os.environ, VFI_CHECK_ROOT=root))
            if r.returncode != 0:
                report("parent:run", False, root=root, error=r.stderr[-2000:])
                return
            outs.append(np.load(p))
        for key in ("rife", "film", "sep", "flavr", "ifrnet", "cain"):
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
    from cfi_b200.engine import IfunetEngine
    import cfi_b200.ifunet_node as UN

    sd = OU.synthetic_state_dict(0)
    for dt in ("float32", "bfloat16"):
        try:
            elem_stages(dt, sd)
        except Exception as e:  # keep going: later stages still tell something
            report(f"elem:{dt}", False, error=repr(e)[:300])

    for use_ref, stage in ((True, "forward_ref"), (False, "forward")):
        for name, cfg in sorted(ifunet_cases().items()):
            if cfg["kind"] != "net":
                continue
            try:
                ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
                e2 = IfunetEngine(case_state_dict(cfg), device=0, dtype="float32")
                e2.set_ref(use_ref)
                x = ifunet_inputs(cfg)[..., :3].permute(0, 3, 1, 2).contiguous().cuda()
                out = e2.forward(x[0:1].contiguous(), x[1:2].contiguous(), cfg["t"], cfg["scale"], cfg["ensemble"])
                torch.cuda.synchronize()
                p = psnr(out.cpu(), ref)
                report(f"{stage}:{name}", p >= 50.0, psnr_db=round(p, 2), max_abs=float((out.cpu() - ref).abs().max()),
                       launches=e2.launch_count())
                e2.close()
            except Exception as e:
                report(f"{stage}:{name}", False, error=repr(e)[:300])

    for name, cfg in sorted(ifunet_cases().items()):
        if cfg["kind"] != "node":
            continue
        try:
            ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
            e3 = IfunetEngine(case_state_dict(cfg), device=0, dtype="float32")
            fr = ifunet_inputs(cfg)
            st = None if cfg["states"] is None else UN.InterpolationStateList(list(cfg["states"][0]), cfg["states"][1])
            (out,) = UN.IFUnet_VFI().vfi("IFUNet.pth", fr, multiplier=cfg["multiplier"], scale_factor=cfg["scale"],
                                         ensemble=cfg["ensemble"], optional_interpolation_states=st, _engine=e3)
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
        e4 = IfunetEngine(sd, device=0)
        x = torch.rand(1, 3, 100, 150, device="cuda")
        for s in (0.25, 0.7, 1.2):
            out = torch.full_like(x, 7.0)
            n0 = e4.launch_count()
            try:
                e4.forward(x, x, 0.5, s, True, out=out)
                refused, msg = False, ""
            except VfiError as err:
                refused, msg = True, str(err)
            torch.cuda.synchronize()
            report(f"refuse:scale_{s}", refused and "the reference raises" in msg and e4.launch_count() == n0
                   and bool((out == 7.0).all()), message=msg[:200])
        e4.close()
    except Exception as e:
        report("refuse", False, error=repr(e)[:300])

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
