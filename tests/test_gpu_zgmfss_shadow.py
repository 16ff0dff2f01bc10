"""-m gpu: every gmops kernel and every soft splat of the GMFSS path per element against float64 on the H100 (the shadow of
tests/gmfss_shadow_util.py): the standalone case matrix, the refusals, and the product schedule (build_gpu_model, union and
base) at the bench's 720p (padded to 768x1280), at 1080p (padded to 1088x1920) and at a golden size.  The per-call bounds
are the gate; each run prints one line per (kernel, variant): calls, worst error / bound and where.

720p and 1080p run different kernels for the same layer (the scale-1 windows hold 12x20 = 240 tokens at 720p and 17x30 =
510 at 1080p; gm_gemm picks 8 / 4 / 2 rows per thread by problem size), so the coverage of each is asserted.  At those
sizes the whole frame and both flows are also compared with the float64 oracle (oracle/gmfss.py, oracle/gmfss_base.py,
fed with the library's own RIFE output), next to the float64 oracle's own response to one fp32 rounding of its inputs and
weights; the numbers are printed (see the comment at the end of the test for why only a floor is asserted there)."""
import os
import sys
import time

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gmfss_shadow_util as SU  # noqa: E402
from make_golden_gmfss import gmfss_cases  # noqa: E402
from oracle import film as OF  # noqa: E402
from oracle import gmfss as OG  # noqa: E402
from oracle import gmfss_base as GB  # noqa: E402
from oracle import gmfss_weights as GW  # noqa: E402
from oracle import rife46 as R  # noqa: E402

pytestmark = pytest.mark.gpu


def _gpu_shadow_ops(pkg):
    from cfi_b200._lib import lib
    return SU.shadow_class()(lib(), torch.device("cuda", 0))


def test_case_matrix_on_h100(pkg):
    t0 = time.time()
    SU.check_matrix(_gpu_shadow_ops(pkg))
    print(f"case matrix: {time.time() - t0:.1f} s")


def test_refusals_on_h100(pkg):
    SU.check_refusals(_gpu_shadow_ops(pkg))


SIZES = {"720p": (720, 1280), "1080p": (1080, 1920), "golden": (96, 128)}


@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("variant", ["union", "base"])
def test_shadowed_product_schedule(pkg, variant, size):
    from cfi_b200.gmfss import build_gpu_model
    t0 = time.time()
    h, w = SIZES[size]
    seed = 0
    sds = (GW if variant == "union" else GB).synthetic_state_dicts(seed)
    fr = OF.synthetic_clip(2, h, w, seed=71).permute(0, 3, 1, 2).contiguous().cuda()
    if size == "golden":   # the 96x128 golden case's own clip
        cfg = gmfss_cases(variant)[("gmfss_" if variant == "union" else "gmfss_base_") + "96x128_t0.5"]
        fr = OF.synthetic_clip(2, h, w, seed=cfg["clip_seed"]).permute(0, 3, 1, 2).contiguous().cuda()
    t = 0.5
    m = build_gpu_model(sds, 0)
    o = SU.shadow(m.o)
    m.splat = SU.shadow_splat(m.splat, o.stats)
    rife_out = []
    if m.rife is not None:
        lib_rife = m.rife
        m.rife = lambda h0, h1, tt: rife_out.append(lib_rife(h0, h1, tt)) or rife_out[-1]   # noqa: E731
    ph, pw = ((h - 1) // 64 + 1) * 64, ((w - 1) // 64 + 1) * 64
    # GMFSS.interpolate, with the state kept for the flow comparison
    i0, i1 = o.new(1, 3, ph, pw), o.new(1, 3, ph, pw)
    o.copy_slice(fr[0:1].contiguous(), i0, 3)
    o.copy_slice(fr[1:2].contiguous(), i1, 3)
    state = m.reuse(i0, i1)
    out = o.copy_slice(m.inference(state, t), o.new(1, 3, h, w), 3)
    torch.cuda.synchronize()
    t_shadow = time.time() - t0
    if m._engine is not None:
        m._engine.close()
    st = o.stats
    print(f"\n{variant} {size} ({h}x{w}, padded {ph}x{pw}): shadowed forward {t_shadow:.1f} s")
    print("\n".join(st.lines(f"{variant} {size} ")))
    assert not st.failures(), st.failures()
    assert st.rows[("splat", "soft")]["calls"] == 8
    gem = st.variants("bmm") | st.variants("linear")
    if size == "1080p":
        assert {"nn8<8>", "nn8<4>", "bt", "nn"} <= gem, gem
        # the 510-token windows: scores on the bt kernel, P V on the generic nn kernel
        assert any(me == "bmm" and v == "bt" and s[1:] == (510, 510) for me, v, s in st.seen)
        assert any(me == "bmm" and v == "nn" and s[1] == 510 for me, v, s in st.seen)
    if size == "720p":
        # the 240-token windows: scores and P V on the 8 x 8-tile kernel
        assert any(me == "bmm" and v.startswith("nn8") and s[1:] == (240, 240) for me, v, s in st.seen)
        assert any(me == "bmm" and v.startswith("nn8") and s[1:] == (240, 128) for me, v, s in st.seen)
    if size == "golden":
        return
    # the whole path against the float64 oracle, fed with the library's RIFE output; and, for scale, the float64 oracle
    # against itself with every weight and both frames perturbed by one fp32 rounding (a relative +-2^-24)
    t1 = time.time()
    g = torch.Generator().manual_seed(5)
    jit = lambda v: v * (1 + SU.U * torch.sign(torch.randn(v.shape, generator=g, dtype=torch.float64))).to(v.device)   # noqa: E731

    def oracle(perturb):
        p_ = jit if perturb else (lambda v: v)
        sd64 = {net: {k: p_(v.to("cuda", torch.float64)) if v.is_floating_point() else v.cuda() for k, v in sd.items()}
                for net, sd in sds.items() if net != "ifnet"}
        with torch.no_grad():
            a0 = F.pad(p_(fr[0:1].double()), (0, pw - w, 0, ph - h))
            a1 = F.pad(p_(fr[1:2].double()), (0, pw - w, 0, ph - h))
            f01, f10, m0, m1, fa, fb = OG.reuse(sd64, a0, a1)
            if variant == "union":
                ref = OG.inference(sd64, a0, a1, f01, f10, m0, m1, fa, fb, t, rife=lambda *_: rife_out[0].double())
            else:
                ref = GB.inference(sd64, a0, a1, f01, f10, m0, m1, fa, fb, t)
        return f01, f10, ref[:, :, :h, :w]

    def dev(tag, A, B):
        e = [(A[i].double() - B[i]).abs() for i in (0, 1)]
        p = R.psnr(A[2].float().cpu(), B[2].float().cpu())
        emax_, emean_ = max(float(x.max()) for x in e), float(sum(x.mean() for x in e)) / 2
        beyond = float(sum((x > 2e-2).double().mean() for x in e)) / 2
        print(f"{variant} {size}: {tag}: flows max {emax_:.3e} px, mean {emean_:.3e} px, {beyond:.1%} of pixels beyond "
              f"2e-2 px; frame PSNR {p:.2f} dB")
        return emax_, emean_, p

    ref64 = oracle(False)
    emax, emean, p = dev("product vs the float64 oracle", (state[0], state[1], out), ref64)
    dev("float64 oracle with its inputs and weights perturbed by one fp32 rounding vs unperturbed", oracle(True), ref64)
    torch.cuda.synchronize()
    print(f"{variant} {size}: oracles {time.time() - t1:.1f} s")
    # GMFlow's global softmax and the transformer amplify fp32 rounding at these sizes.  Measured on an H100 (700 W): one fp32
    # rounding of the float64 oracle's own inputs and weights moves its flows by up to 0.2-0.6 px (0.7-10 % of the pixels
    # beyond 2e-2 px, 40-46 dB); the product, which rounds in every operation, lands 1.5-3.4 px max / 0.014-0.029 px mean
    # from it (34-38 dB) while every call stays inside its bound.  So the golden criteria (50 dB, 2e-2 px max) cannot hold
    # against float64 here; the per-call bounds are the gate, and this is only a floor under the measured whole path.
    assert p >= 30.0 and emean <= 0.1, (p, emean, emax)
