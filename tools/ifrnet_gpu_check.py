#!/usr/bin/env python
"""IFRNet on the GPU, checked stage by stage (run on an H100; tests/test_gpu_zifrnet.py runs it in a subprocess).

    python tools/ifrnet_gpu_check.py [--parent-src DIR]

Stages, each reported as one JSON line {"stage": ..., "ok": ..., ...}; exit code 0 only if every stage passed:
  conv:<dtype>:<kind>   one streamconv layer of every kind IFRNet uses, with the IFRNet epilogue (per-channel PReLU,
                        residual before it, fp32 columns): a 3x3 conv, a stride-2 conv over the space-to-depth copy, a
                        ResBlock side-channel conv, conv5 on two sources with the residual, the four ConvT phases; on
                        random 16-bit inputs in the padded channel layout: wgmma kernel vs the CUDA-core checker (same
                        packed weights) and the checker vs torch conv2d / conv_transpose2d, fp16 and bf16 operands
  conv1080              pyramid1.1 at the 1080p geometry (multiplier 2: 2 x 272 x 480), wgmma vs checker
  forward_ref / forward both variants through libvfi_b200.so on the checker / on the wgmma kernel vs the unmodified
                        reference's output (tests/golden/ifrnet_*.npz; the t = 1/3 cases run the decoder inputs on grids
                        that differ from the encoder levels they warp): PSNR >= 50 dB
  node                  IFRNet_VFI.vfi vs the unmodified reference node (tests/golden/ifrnet_node_*.npz): interpolated
                        frames PSNR >= 50 dB, pass-through frames bit-exact
  parent:film / parent:sepconv / parent:flavr   with --parent-src (a checkout of the parent commit): outputs on seeded
                        inputs bit-identical between this library and the parent's, built in a temp directory
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

from make_golden_ifrnet import case_state_dict, ifrnet_cases, ifrnet_inputs  # noqa: E402
from oracle import film as OF  # noqa: E402
from oracle import ifrnet as OI  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
RESULTS = []


def report(stage, ok, **kw):
    row = dict(stage=stage, ok=bool(ok), **kw)
    RESULTS.append(row)
    print(json.dumps(row), flush=True)


def psnr(a, b):
    mse = float(((a.double() - b.double()) ** 2).mean())
    return 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)


# ---- the channel layouts of ifrnet.cu (physical channel -> logical, -1 = padding)
def up(v, a):
    return (v + a - 1) // a * a


def map_plain(c):
    return [j if j < c else -1 for j in range(up(c, 64))]


def map_split(c, s):
    m = up(c - s, 64)
    out = [-1] * (m + up(s, 64))
    for j in range(c - s):
        out[j] = j
    for i in range(s):
        out[m + i] = c - s + i
    return out


def to_phys(x, m):
    """[..., C logical] -> [..., len(m)] with zeros in the padding channels"""
    idx = torch.tensor([j if j >= 0 else 0 for j in m])
    keep = torch.tensor([1.0 if j >= 0 else 0.0 for j in m], dtype=x.dtype)
    return x[..., idx] * keep


def to_log(x, m, c):
    """[..., len(m)] -> [..., c]"""
    pos = [0] * c
    for j, v in enumerate(m):
        if v >= 0:
            pos[v] = j
    return x[..., pos]


def conv_stage(dt, kind, sd, eng, B=2, H=18, W=22):
    """One layer kind of IFRNet-S; the torch reference uses the fp16/bf16-rounded inputs and weights."""
    g = torch.Generator().manual_seed(sum(map(ord, kind)))
    td = torch.float16 if dt == "float32" else torch.bfloat16
    q = lambda t: t.to(td).float()  # noqa: E731
    rnd = lambda *s: q(torch.rand(*s, generator=g) - 0.5)  # noqa: E731
    nchw = lambda x: x.permute(0, 3, 1, 2)  # noqa: E731
    nhwc = lambda x: x.permute(0, 2, 3, 1)  # noqa: E731
    cu = lambda x: x.to(td).cuda().contiguous()  # noqa: E731

    def both(fn):
        outs = []
        for impl in (1, 0):
            outs.append(fn(impl))
            torch.cuda.synchronize()
        return outs

    def plain_out(layer, src0, p0, src1, p1, n_pitch, res=None, B_=B, H_=H, W_=W):
        def run(impl):
            out = torch.full((B_, H_, W_, n_pitch), float("nan"), dtype=td, device="cuda")
            eng.debug_conv(layer, src0, p0, src1, p1, out, n_pitch, B_, H_, W_, impl=impl, res=res)
            return out.float().cpu()
        return both(run)

    if kind == "conv3_prelu":              # pyramid1.1: 24 -> 24, per-channel PReLU
        p = "encoder.pyramid1.1."
        x = rnd(B, H, W, 24)
        ref_k, tc = plain_out(0, cu(to_phys(x, map_plain(24))), 64, None, 0, 64)
        ref_k, tc = ref_k[..., :24], tc[..., :24]
        y = nhwc(F.prelu(F.conv2d(nchw(x), q(sd[p + "0.weight"]), sd[p + "0.bias"], padding=1), sd[p + "1.weight"]))
    elif kind == "stride2_s2d":             # pyramid2.0: 24 -> 36, stride 2 as a 2x2 conv over the space-to-depth copy
        p = "encoder.pyramid2.0."
        full = rnd(B, 2 * H, 2 * W, 24)
        s2d = torch.zeros(B, H, W, 128)
        for qd in range(4):
            s2d[..., qd * 24:(qd + 1) * 24] = full[:, qd >> 1::2, qd & 1::2, :]
        ref_k, tc = plain_out(1, cu(s2d), 128, None, 0, 64)
        ref_k, tc = ref_k[..., :36], tc[..., :36]
        y = nhwc(F.prelu(F.conv2d(nchw(full), q(sd[p + "0.weight"]), sd[p + "0.bias"], stride=2, padding=1),
                         sd[p + "1.weight"]))
    elif kind == "side_conv":               # decoder4 ResBlock conv2: reads the 24 side channels at 128 of a 192 tensor
        p = "decoder4.convblock.1.conv2."
        x = rnd(B, H, W, 144)
        xp = cu(to_phys(x, map_split(144, 24)))
        ref_k, tc = plain_out(12, xp[..., 128:], 192, None, 0, 64)
        ref_k, tc = ref_k[..., :24], tc[..., :24]
        y = nhwc(F.prelu(F.conv2d(nchw(x[..., 120:]), q(sd[p + "0.weight"]), sd[p + "0.bias"], padding=1),
                         sd[p + "1.weight"]))
    elif kind == "conv5_two_sources_residual":  # decoder4 conv5: cat(main slice of b, side tensor) + x, then PReLU
        p = "decoder4.convblock.1."
        b, side, x = rnd(B, H, W, 144), rnd(B, H, W, 24), rnd(B, H, W, 144)
        m = map_split(144, 24)
        bp = cu(to_phys(b, m))
        sp = cu(to_phys(side, map_plain(24)))
        xr = cu(to_phys(x, m))
        ref_k, tc = plain_out(15, bp, 192, sp, 64, 192, res=xr)
        ref_k, tc = to_log(ref_k, m, 144), to_log(tc, m, 144)
        xin = torch.cat([b[..., :120], side], -1)
        y = nhwc(F.prelu(nchw(x) + F.conv2d(nchw(xin), q(sd[p + "conv5.weight"]), sd[p + "conv5.bias"], padding=1),
                         sd[p + "prelu.weight"]))
    elif kind == "convt_phases":            # decoder4 ConvTranspose2d(144, 58, 4, 2, 1): flows fp32, ft_ 16-bit
        p = "decoder4.convblock.2."
        x = rnd(1, H, W, 144)
        xp = cu(to_phys(x, map_split(144, 24)))
        yt = nhwc(F.conv_transpose2d(nchw(x), q(sd[p + "weight"]), sd[p + "bias"], stride=2, padding=1))

        def run(impl):
            o16 = torch.full((1, H, W, 4 * 64), float("nan"), dtype=td, device="cuda")
            o32 = torch.full((1, H, W, 16), float("nan"), dtype=torch.float32, device="cuda")
            for ph in range(4):
                eng.debug_conv(16 + ph, xp, 192, None, 0, o16[..., ph * 64:], 256, 1, H, W, impl=impl,
                               out_f32=o32[..., ph * 4:], f32_pitch=16)
            o16, o32 = o16.float().cpu(), o32.cpu()
            full = torch.zeros(1, 2 * H, 2 * W, 58)
            for ph in range(4):
                full[:, ph >> 1::2, ph & 1::2, 0:4] = o32[..., ph * 4:ph * 4 + 4]
                full[:, ph >> 1::2, ph & 1::2, 4:] = o16[..., ph * 64 + 8:ph * 64 + 62]
            return full
        ref_k, tc = both(run)
        y = yt
    else:
        raise ValueError(kind)
    scale = float(ref_k.abs().max()) + 1e-6
    err_tc = float((tc - ref_k).abs().max()) / scale
    err_t = float((ref_k - y).abs().max()) / (float(y.abs().max()) + 1e-6)
    nan = int(torch.isnan(tc).sum() + torch.isnan(ref_k).sum())
    tol = 4e-3 if dt == "float32" else 2e-2
    report(f"conv:{dt}:{kind}", err_tc <= (4e-3 if dt == "float32" else 1e-2) and err_t <= tol and nan == 0,
           rel_err_tc_vs_checker=err_tc, rel_err_checker_vs_torch=err_t, nan=nan)


def conv1080_stage(eng):
    """pyramid1.1 at 1080p, multiplier 2: both frames at 272 x 480 (2 x 34 x 60 tiles)."""
    B, H, W = 2, 272, 480
    g = torch.Generator().manual_seed(5)
    x = torch.zeros(B, H, W, 64)
    x[..., :24] = torch.rand(B, H, W, 24, generator=g) - 0.5
    xd = x.half().cuda()
    outs = []
    for impl in (1, 0):
        out = torch.full((B, H, W, 64), float("nan"), dtype=torch.float16, device="cuda")
        eng.debug_conv(0, xd, 64, None, 0, out, 64, B, H, W, impl=impl)
        torch.cuda.synchronize()
        outs.append(out.float().cpu())
    ref_k, tc = outs
    err = float((tc - ref_k).abs().max()) / (float(ref_k.abs().max()) + 1e-6)
    report("conv1080:pyramid1.1", err <= 4e-3 and not torch.isnan(tc).any(), rel_err_tc_vs_checker=err,
           plan=eng.layer_plan(0))


def parent_outputs(path):
    """FILM, Sepconv and FLAVR on seeded inputs with this process's library -> npz (for the parent comparison)."""
    import __graft_entry__ as ge
    ge.load_package()
    from cfi_b200.engine import FilmEngine, FlavrEngine, SepconvEngine
    from oracle import flavr as OV
    from oracle import sepconv as OS
    fr = OF.synthetic_clip(5, 72, 104, seed=61).cuda()
    film = FilmEngine(OF.synthetic_state_dict(1, 2.0), device=0, dtype="float32").forward(fr, [0, 1], [1, 2]).cpu().numpy()
    sep = SepconvEngine(OS.synthetic_state_dict(5), device=0).forward(fr, [0, 1], [1, 2]).cpu().numpy()
    flavr = FlavrEngine(OV.synthetic_state_dict(0, "4x"), device=0).forward(fr.contiguous(), [0, 1]).cpu().numpy()
    np.savez(path, film=film, sep=sep, flavr=flavr)


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
            r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "ifrnet_gpu_check.py"), "--parent-outputs", p],
                               cwd=root, capture_output=True, text=True, env=dict(os.environ, VFI_CHECK_ROOT=root))
            if r.returncode != 0:
                report("parent:run", False, root=root, error=r.stderr[-2000:])
                return
            outs.append(np.load(p))
        for key in ("film", "sep", "flavr"):
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
    from cfi_b200.engine import IfrnetEngine
    import cfi_b200.ifrnet_node as IN

    sd = OI.synthetic_state_dict("S", 0)
    kinds = ["conv3_prelu", "stride2_s2d", "side_conv", "conv5_two_sources_residual", "convt_phases"]
    for dt in ("float32", "bfloat16"):
        eng = IfrnetEngine(sd, device=0, dtype=dt)
        for kind in kinds:
            try:
                conv_stage(dt, kind, sd, eng)
            except Exception as e:  # keep going: later stages still tell something
                report(f"conv:{dt}:{kind}", False, error=repr(e)[:300])
        if dt == "float32":
            try:
                conv1080_stage(eng)
            except Exception as e:
                report("conv1080:pyramid1.1", False, error=repr(e)[:300])
        eng.close()

    for use_ref, stage in ((True, "forward_ref"), (False, "forward")):
        for name, cfg in sorted(ifrnet_cases().items()):
            if cfg["kind"] != "net":
                continue
            try:
                ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
                e2 = IfrnetEngine(case_state_dict(cfg), device=0, dtype="float32")
                e2.set_ref(use_ref)
                x = ifrnet_inputs(cfg)[..., :3].permute(0, 3, 1, 2).contiguous().cuda()
                out = e2.forward(x[0:1].contiguous(), x[1:2].contiguous(), cfg["t"], cfg["embt"])
                torch.cuda.synchronize()
                p = psnr(out.cpu(), ref)
                report(f"{stage}:{name}", p >= 50.0 and e2.variant == cfg["variant"], psnr_db=round(p, 2),
                       launches=e2.launch_count())
                e2.close()
            except Exception as e:
                report(f"{stage}:{name}", False, error=repr(e)[:300])

    for name, cfg in sorted(ifrnet_cases().items()):
        if cfg["kind"] != "node":
            continue
        try:
            ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
            e3 = IfrnetEngine(case_state_dict(cfg), device=0, dtype="float32")
            fr = ifrnet_inputs(cfg)
            st = None if cfg["states"] is None else IN.InterpolationStateList(list(cfg["states"][0]), cfg["states"][1])
            (out,) = IN.IFRNet_VFI().vfi(cfg["ckpt"], fr, multiplier=cfg["multiplier"], scale_factor=cfg["scale_factor"],
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
