"""Every gmops kernel of the GMFSS path per element against float64, on the CPU: csrc/gmops.cu compiled for the host
(tests/host_emu/gmops_emu.cpp) under the float64 shadow of tests/gmfss_shadow_util.py.

- The float64 references are pinned to the oracle functions they restate (the oracle in its float64 mode), so a wrong
  reference cannot agree with a wrong kernel.
- The standalone case matrix: every kernel variant at the shapes and edges where such kernels go wrong; every element
  within its a-priori bound.
- The product schedule (GMFSS.interpolate) of one union and one base golden case, every call shadowed.
- The launchers' refusals.
The same matrix and schedule run on the H100 in tests/test_gpu_zgmfss_shadow.py."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gmfss_shadow_util as SU  # noqa: E402
from make_golden_gmfss import gmfss_cases  # noqa: E402
from oracle import film as OF  # noqa: E402
from oracle import gmflow as GF  # noqa: E402
from oracle import gmfss as OG  # noqa: E402
from oracle import gmfss_base as GB  # noqa: E402
from oracle import gmfss_weights as GW  # noqa: E402
from oracle import ops_ref  # noqa: E402
from oracle import rife46 as R  # noqa: E402

CUDA_INC = "/usr/local/cuda/include"
D = torch.float64


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not (shutil.which("g++") and os.path.exists(os.path.join(CUDA_INC, "cuda_fp16.h"))):
        pytest.skip("g++ / CUDA headers not available")
    so = str(tmp_path_factory.mktemp("emu") / "libgmopsemu.so")
    src = os.path.join(ROOT, "tests", "host_emu", "gmops_emu.cpp")
    r = subprocess.run(["g++", "-O2", "-std=c++20", "-shared", "-fPIC", "-pthread", "-I" + CUDA_INC, "-o", so, src] +
                       os.environ.get("VFI_EMU_CXXFLAGS", "").split(), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(so)


def _shadow_ops(lib):
    return SU.shadow_class()(lib, torch.device("cpu"))


def _close(a, b, tol=1e-12):
    return float((a - b).abs().max()) <= tol * max(1.0, float(b.abs().max()))


# ----------------------------------------------------------------------------------------------- references pinned
def test_references_match_the_float64_oracle():
    g = torch.Generator().manual_seed(3)
    rn = lambda *s, scale=1.0: torch.randn(*s, generator=g, dtype=D) * scale   # noqa: E731
    # window split with the cyclic shift
    b, h, w, c, k = 2, 12, 16, 5, 4
    tok = rn(b, h * w, c)
    rolled = torch.roll(tok.view(b, h, w, c), shifts=(-1, -2), dims=(1, 2))
    assert torch.equal(SU._window_split(tok, b, h, w, c, k, 1, 2), GF._windows_last(rolled, k).reshape(b * k * k, -1, c))
    assert torch.equal(SU._window_merge(SU._window_split(tok, b, h, w, c, k, 1, 2), b, h, w, c, k, 1, 2), tok)
    # position embedding inside the windows
    f0, f1 = rn(1, 16, 8, 12), rn(1, 16, 8, 12)
    for k in (1, 2, 4):
        a0, _ = GF.add_position(f0, f1, k)
        assert _close(f0 + SU.ref_position(f0.shape, k, f0.device)[0], a0), k
    # local correlation softmax, R = 1..4, also on planes smaller than the window
    for r in (1, 2, 3, 4):
        for hh, ww in ((8, 12), (2, 3)):
            a, bb = rn(1, 16, hh, ww), rn(1, 16, hh, ww)
            ref = GF.local_match(a, bb, r)
            got = SU.ref_local_match(a, bb, r)
            assert _close(got[0][0], ref[:, 0]) and _close(got[1][0], ref[:, 1]), (r, hh, ww)
    # radius-1 propagation (the oracle projects the tokens itself)
    cc = 16
    sd = {"feature_flow_attn.q_proj.weight": rn(cc, cc, scale=0.3), "feature_flow_attn.q_proj.bias": rn(cc),
          "feature_flow_attn.k_proj.weight": rn(cc, cc, scale=0.3), "feature_flow_attn.k_proj.bias": rn(cc)}
    feat, flow = rn(2, cc, 6, 9), rn(2, 2, 6, 9, scale=3.0)
    x = feat.flatten(2).transpose(1, 2)
    q = F.linear(x, sd["feature_flow_attn.q_proj.weight"], sd["feature_flow_attn.q_proj.bias"])
    kk = F.linear(x, sd["feature_flow_attn.k_proj.weight"], sd["feature_flow_attn.k_proj.bias"])
    ref = GF.propagate(sd, feat, flow, 1)
    got = SU.ref_local_prop(q, kk, flow)
    assert _close(got[0][0], ref[:, 0]) and _close(got[1][0], ref[:, 1])
    # convex up-sampling (the oracle computes the mask with the upsampler convs)
    sd = {"upsampler.0.weight": rn(32, cc + 2, 3, 3, scale=0.1), "upsampler.0.bias": rn(32),
          "upsampler.2.weight": rn(9 * 16, 32, 1, 1, scale=0.2), "upsampler.2.bias": rn(9 * 16)}
    mask = F.conv2d(F.relu(F.conv2d(torch.cat((flow, feat), 1), sd["upsampler.0.weight"], sd["upsampler.0.bias"], padding=1)),
                    sd["upsampler.2.weight"], sd["upsampler.2.bias"])
    ref = GF.upsample_convex(sd, flow, feat)
    got = SU.ref_convex_up(mask, flow, 4)
    assert _close(got[0][0], ref[:, 0]) and _close(got[1][0], ref[:, 1])
    # warps: flow_warp, backwarp, and the forward-backward consistency flags
    img = torch.rand(2, 3, 9, 13, generator=g, dtype=D)
    fl = rn(2, 2, 9, 13, scale=6.0)
    assert _close(SU.ref_warp(img, fl)[0], OG._flow_warp(img, fl))
    assert _close(SU.ref_warp(img, fl)[0], OG.backwarp(img, fl), 1e-10)
    fb = rn(2, 2, 9, 13, scale=6.0)
    occ_f, occ_b = OG.fb_consistency(fl, fb)
    (mf, _), (mb, _) = SU.ref_fb_margins(fl, fb)
    assert torch.equal((mf > 0).to(D), occ_f) and torch.equal((mb > 0).to(D), occ_b)
    # the soft splat (addeps)
    xs, met = rn(2, 4, 9, 13), rn(2, 1, 9, 13)
    ref = ops_ref.softsplat(xs, fl, met, "soft")
    assert ref.dtype == D
    assert _close(SU.splat_reference(xs, fl, met)[0], ref, 1e-10)


def test_float64_oracle_on_a_golden_case():
    """the oracle's float64 mode runs the whole model and lands on the golden (made in fp32 by the reference)"""
    name = "gmfss_96x128_t0.5"
    cfg = gmfss_cases()[name]
    g = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    sds = {net: {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}
           for net, sd in GW.synthetic_state_dicts(cfg["seed"]).items()}
    fr = OF.synthetic_clip(2, cfg["h"], cfg["w"], seed=cfg["clip_seed"]).permute(0, 3, 1, 2).double()
    h, w = cfg["h"], cfg["w"]
    ph, pw = ((h - 1) // 64 + 1) * 64, ((w - 1) // 64 + 1) * 64
    with torch.no_grad():
        i0, i1 = F.pad(fr[0:1], (0, pw - w, 0, ph - h)), F.pad(fr[1:2], (0, pw - w, 0, ph - h))
        h0 = F.interpolate(i0, scale_factor=0.5, mode="bilinear", align_corners=False)
        h1 = F.interpolate(i1, scale_factor=0.5, mode="bilinear", align_corners=False)
        f01 = GF.gmflow(sds["flownet"], h0, h1)
        rife = lambda a, b, t: R.ifnet46_forward(GW.synthetic_state_dicts(cfg["seed"])["ifnet"], a.float(), b.float(),  # noqa: E731
                                                 torch.full((1, 1, 1, 1), float(t)), (8, 4, 2, 1)).double()
        out = OG.interpolate(sds, fr[0:1], fr[1:2], cfg["t"], rife=rife)
    assert f01.dtype == D and out.dtype == D
    e = float((f01 - torch.from_numpy(g["flow01"]).double()).abs().max())
    p = R.psnr(out.float(), torch.from_numpy(g["out"]))
    print(f"{name}: float64 oracle flow within {e:.2e} px, frame PSNR {p:.1f} dB of the fp32 golden")
    assert e <= 2e-2 and p >= 50.0


# ----------------------------------------------------------------------------------------------- standalone matrix
def test_case_matrix_on_the_host_build(emu):
    SU.check_matrix(_shadow_ops(emu))


def test_refusals_on_the_host_build(emu):
    SU.check_refusals(_shadow_ops(emu))


# ----------------------------------------------------------------------------------------------- the golden schedules
@pytest.mark.parametrize("variant,name", [("union", "gmfss_96x128_t0.5"), ("base", "gmfss_base_70x100_t0.3")])
def test_shadowed_schedule_on_the_host_build(emu, variant, name):
    """GMFSS.interpolate of a golden case with every gmops call and every splat checked against float64"""
    import __graft_entry__ as ge
    ge.load_package()
    from cfi_b200.gmfss import GMFSS
    cfg = gmfss_cases(variant)[name]
    sds = (GW if variant == "union" else GB).synthetic_state_dicts(cfg["seed"])
    fr = OF.synthetic_clip(2, cfg["h"], cfg["w"], seed=cfg["clip_seed"]).permute(0, 3, 1, 2).contiguous()
    o = _shadow_ops(emu)
    splat = SU.shadow_splat(lambda x, fl, z: ops_ref.softsplat(x, fl, z, "soft"), o.stats)
    rife = None
    if variant == "union":
        rife = lambda h0, h1, t: R.ifnet46_forward(sds["ifnet"], h0, h1, torch.full((h0.shape[0], 1, 1, 1), float(t)),  # noqa: E731
                                                   (8, 4, 2, 1))
    m = GMFSS(sds, o, splat=splat, rife=rife)
    out = m.interpolate(fr[0:1].contiguous(), fr[1:2].contiguous(), cfg["t"])
    print("\n" + "\n".join(o.stats.lines(f"{name} ")))
    assert out.shape == (1, 3, cfg["h"], cfg["w"])
    assert not o.stats.failures(), o.stats.failures()
    assert o.stats.rows[("splat", "soft")]["calls"] == 8
