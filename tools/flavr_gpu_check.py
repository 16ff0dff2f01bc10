#!/usr/bin/env python
"""FLAVR on the GPU, checked stage by stage (run on an H100; tests/test_gpu_zflavr.py runs it in a subprocess).

    python tools/flavr_gpu_check.py [--quick] [--parent-src DIR]

Stages, each reported as one JSON line {"stage": ..., "ok": ..., ...}; exit code 0 only if every stage passed:
  conv:<dtype>:<kind>   one streamconv layer of every kind FLAVR uses (3x3x3 on two sources, stride 2 over the
                        space-to-depth copy, 1x1x1 downsample, the four phases of a transposed conv, the kt = 4 fuse) on
                        random 16-bit inputs: wgmma kernel vs the CUDA-core checker (same packed weights) and the checker
                        vs torch conv3d / conv_transpose3d / conv2d with the layer's weights, fp16 and bf16 operands
  conv1080:<kind>       the same at the 1080p geometry (each persistent CTA walks many tiles), wgmma vs checker
  forward_ref / forward the model through libvfi_b200.so on the checker / on the wgmma kernel vs the unmodified
                        reference's output (tests/golden/flavr_*.npz): PSNR >= 50 dB
  node                  FLAVR_VFI.vfi vs the unmodified reference node (tests/golden/flavr_node_*.npz)
  parent:film / parent:sepconv   with --parent-src (a checkout of the parent commit): FILM and Sepconv on seeded inputs,
                        bit-identical between this library and the parent's, built in a temp directory
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

from make_golden_flavr import flavr_cases, flavr_inputs  # noqa: E402
from oracle import film as OF  # noqa: E402
from oracle import flavr as OV  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
RESULTS = []
T = 4


def report(stage, ok, **kw):
    row = dict(stage=stage, ok=bool(ok), **kw)
    RESULTS.append(row)
    print(json.dumps(row), flush=True)


def psnr(a, b):
    mse = float(((a.double() - b.double()) ** 2).mean())
    return 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)


def to_ncthw(x, S):
    """[S*T, H, W, C] -> [S, C, T, H, W] float32 CPU"""
    n, h, w, c = x.shape
    return x.float().cpu().view(S, n // S, h, w, c).permute(0, 4, 1, 2, 3)


def s2d(x):
    """[n, H, W, C] -> [n, H/2, W/2, 4 C], phase (y & 1) * 2 + (x & 1) at channel phase * C"""
    n, h, w, c = x.shape
    return x.view(n, h // 2, 2, w // 2, 2, c).permute(0, 1, 3, 2, 4, 5).reshape(n, h // 2, w // 2, 4 * c).contiguous()


def run_layer(eng, layer, x0, x1, n_out, S, H, W, out_pitch=None, T_out=T):
    outs = []
    for impl in (1, 0):
        out = torch.full((S * T_out, H, W, out_pitch or n_out), float("nan"), dtype=x0.dtype, device="cuda")
        eng.debug_conv(layer, x0, x1, out, S, H, W, impl=impl)
        torch.cuda.synchronize()
        outs.append(out.float().cpu())
    return outs


def conv_stage(dt, kind, sd, eng, S=2, H=18, W=22):
    """One layer kind; the torch reference is computed from the fp16/bf16-rounded inputs and weights."""
    g = torch.Generator().manual_seed(sum(map(ord, kind)))
    td = torch.float16 if dt == "float32" else torch.bfloat16
    rnd = lambda *s: (torch.rand(*s, generator=g) - 0.5).to(td).cuda()  # noqa: E731
    q = lambda t: t.to(td).float()  # noqa: E731
    if kind == "conv333_two_sources":   # decoder 3: cat(dx1 64, x1 64) -> 64, 3x3x3
        layer, p = 52, "decoder.3.conv.0."
        a, b = rnd(S * T, H, W, 64), rnd(S * T, H, W, 64)
        ref_k, tc = run_layer(eng, layer, a, b, 64, S, H, W)
        x = torch.cat([to_ncthw(a, S), to_ncthw(b, S)], 1)
        y = F.conv3d(x, q(sd[p + "weight"]), sd[p + "bias"], padding=1)
    elif kind == "conv333_512_splits":  # layer4 block 1 conv2: 512 -> 512, four output-channel splits
        layer, p = 34, "encoder.layer4.1.conv2.0."
        a = rnd(S * T, H, W, 512)
        ref_k, tc = run_layer(eng, layer, a, None, 512, S, H, W)
        bias = sd.get(p + "bias")
        y = F.conv3d(to_ncthw(a, S), q(sd[p + "weight"]), bias, padding=1)
    elif kind == "stride2_s2d":          # layer2 block 0 conv1: 64 -> 128, stride (1,2,2), ReLU epilogue
        layer, p = 10, "encoder.layer2.0.conv1.0."
        full = rnd(S * T, 2 * H, 2 * W, 64)
        ref_k, tc = run_layer(eng, layer, s2d(full), None, 128, S, H, W)
        y = F.relu(F.conv3d(to_ncthw(full, S), q(sd[p + "weight"]), sd.get(p + "bias"), stride=(1, 2, 2), padding=1))
    elif kind == "downsample111":        # layer2 block 0 downsample: phase-(0,0) slice of the space-to-depth copy
        layer, p = 12, "encoder.layer2.0.downsample.0."
        full = rnd(S * T, 2 * H, 2 * W, 64)
        ref_k, tc = [], None
        xs = s2d(full)
        for impl in (1, 0):
            out = torch.full((S * T, H, W, 128), float("nan"), dtype=td, device="cuda")
            eng.debug_conv(layer, xs, None, out, S, H, W, impl=impl, pitch0=256)
            torch.cuda.synchronize()
            ref_k.append(out.float().cpu())
        ref_k, tc = ref_k
        y = F.conv3d(to_ncthw(full, S), q(sd[p + "weight"]), stride=(1, 2, 2))
    elif kind == "transposed_phases":    # decoder 4: ConvTranspose3d(128, 64, (3,4,4), (1,2,2), 1) on cat(dx0, x0)
        a, b = rnd(S * T, H, W, 64), rnd(S * T, H, W, 64)
        x = torch.cat([to_ncthw(a, S), to_ncthw(b, S)], 1)
        p = "decoder.4.upconv.0."
        yt = F.conv_transpose3d(x, q(sd[p + "weight"]), sd[p + "bias"], stride=(1, 2, 2), padding=1)
        ks, ts, ys = [], [], []
        for ph in range(4):
            rk, tt = run_layer(eng, 56 + ph, a, b, 64, S, H, W)
            ks.append(rk)
            ts.append(tt)
            ys.append(yt[..., ph >> 1::2, ph & 1::2])
        ref_k, tc, y = torch.cat(ks, -1), torch.cat(ts, -1), torch.cat(ys, 1)
    elif kind == "fuse_kt4":             # feature_fuse: cat(unbind(T)) + 1x1 conv = kt 4, T_out 1, LeakyReLU
        a = rnd(S * T, H, W, 64)
        ref_k, tc = run_layer(eng, 60, a, None, 64, S, H, W, T_out=1)
        x = to_ncthw(a, S)
        x2 = torch.cat(torch.unbind(x, 2), 1)
        y = F.leaky_relu(F.conv2d(x2, q(sd["feature_fuse.conv.0.weight"])), 0.2).unsqueeze(2)
    else:
        raise ValueError(kind)
    y = y.permute(0, 2, 3, 4, 1).reshape(ref_k.shape[0], H, W, -1) if y.dim() == 5 else y
    scale = float(ref_k.abs().max()) + 1e-6
    err_tc = float((tc - ref_k).abs().max()) / scale
    err_t = float((ref_k - y).abs().max()) / (float(y.abs().max()) + 1e-6)
    nan = int(torch.isnan(tc).sum() + torch.isnan(ref_k).sum())
    tol = 4e-3 if dt == "float32" else 2e-2
    report(f"conv:{dt}:{kind}", err_tc <= (4e-3 if dt == "float32" else 1e-2) and err_t <= tol and nan == 0, rel_err_tc_vs_checker=err_tc,
           rel_err_checker_vs_torch=err_t, nan=nan)


def conv1080_stage(eng):
    """layer1 conv2 (3x3x3, 64 -> 64) at the 1080p H/2 geometry (544 x 960, four planes: 16320 tiles)."""
    S, H, W = 1, 544, 960
    g = torch.Generator().manual_seed(5)
    a = (torch.rand(S * T, H, W, 64, generator=g) - 0.5).half().cuda()
    ref_k, tc = run_layer(eng, 1, a, None, 64, S, H, W)
    err = float((tc - ref_k).abs().max()) / (float(ref_k.abs().max()) + 1e-6)
    report("conv1080:conv333", err <= 4e-3 and not torch.isnan(tc).any(), rel_err_tc_vs_checker=err,
           plan=eng.layer_plan(1))


def film_sep_outputs(path):
    """FILM and Sepconv on seeded inputs with this process's library -> npz (for the parent comparison)."""
    import __graft_entry__ as ge
    ge.load_package()
    from cfi_b200.engine import FilmEngine, SepconvEngine
    from oracle import sepconv as OS
    fr = OF.synthetic_clip(3, 72, 104, seed=61).cuda()
    fe = FilmEngine(OF.synthetic_state_dict(1, 2.0), device=0, dtype="float32")
    film = fe.forward(fr, [0, 1], [1, 2]).cpu().numpy()
    se = SepconvEngine(OS.synthetic_state_dict(5), device=0)
    sep = se.forward(fr, [0, 1], [1, 2]).cpu().numpy()
    np.savez(path, film=film, sep=sep)


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
            r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "flavr_gpu_check.py"), "--film-sep", p],
                               cwd=root, capture_output=True, text=True, env=dict(os.environ, VFI_CHECK_ROOT=root))
            if r.returncode != 0:
                report("parent:run", False, root=root, error=r.stderr[-2000:])
                return
            outs.append(np.load(p))
        for key in ("film", "sep"):
            a, b = outs[0][key], outs[1][key]
            report(f"parent:{key}", a.shape == b.shape and a.tobytes() == b.tobytes(), shape=list(a.shape),
                   max_abs_diff=float(np.abs(a - b).max()))


def main():
    quick = "--quick" in sys.argv
    if "--film-sep" in sys.argv:
        root = os.environ.get("VFI_CHECK_ROOT", ROOT)
        sys.path.insert(0, root)
        film_sep_outputs(sys.argv[sys.argv.index("--film-sep") + 1])
        return 0
    import __graft_entry__ as ge
    ge.load_package()
    from cfi_b200.engine import FlavrEngine
    import cfi_b200.flavr_node as FN

    sd = OV.synthetic_state_dict(0, "4x")  # encoder biases present
    kinds = ["conv333_two_sources", "stride2_s2d", "downsample111", "transposed_phases", "fuse_kt4", "conv333_512_splits"]
    for dt in ("float32", "bfloat16"):
        eng = FlavrEngine(sd, device=0, dtype=dt)
        for kind in kinds:
            try:
                conv_stage(dt, kind, sd, eng)
            except Exception as e:  # keep going: later stages still tell something
                report(f"conv:{dt}:{kind}", False, error=repr(e)[:300])
        if dt == "float32":
            try:
                conv1080_stage(eng)
            except Exception as e:
                report("conv1080:conv333", False, error=repr(e)[:300])
        eng.close()

    for use_ref, stage in ((True, "forward_ref"), (False, "forward")):
        for name, cfg in sorted(flavr_cases().items()):
            if cfg["kind"] != "net":
                continue
            try:
                gold = np.load(os.path.join(GOLD, name + ".npz"))
                e2 = FlavrEngine(OV.synthetic_state_dict(cfg["seed"], cfg["variant"]), device=0, dtype="float32")
                e2.set_ref(use_ref)
                fr = flavr_inputs(cfg).cuda().contiguous()
                out = e2.forward(fr, [0])
                torch.cuda.synchronize()
                ref = torch.from_numpy(gold["out"]).permute(0, 2, 3, 1)
                p = psnr(out.cpu(), ref)
                report(f"{stage}:{name}", p >= 50.0, psnr_db=round(p, 2), launches=e2.launch_count(),
                       n_outputs=e2.n_outputs, enc_bias=e2.enc_bias)
                e2.close()
            except Exception as e:
                report(f"{stage}:{name}", False, error=repr(e)[:300])

    for name, cfg in sorted(flavr_cases().items()):
        if cfg["kind"] != "node" or (quick and name != "flavr_node_skip_first"):
            continue
        try:
            ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
            e3 = FlavrEngine(OV.synthetic_state_dict(cfg["seed"], cfg["variant"]), device=0, dtype="float32")
            st = None if cfg["states"] is None else FN.InterpolationStateList(list(cfg["states"][0]), cfg["states"][1])
            import warnings
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                (out,) = FN.FLAVR_VFI().vfi(cfg["ckpt"], flavr_inputs(cfg), multiplier=cfg["multiplier"],
                                            duplicate_first_last_frames=cfg["dup"], optional_interpolation_states=st,
                                            _engine=e3)
            p = psnr(out, ref)
            report(f"node:{name}", out.shape == ref.shape and p >= 50.0, psnr_db=round(p, 2), shape=list(out.shape))
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
