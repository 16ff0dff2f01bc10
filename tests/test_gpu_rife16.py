"""-m gpu: the whole RIFE path on the H100 (wgmma layers) against the 16-bit-faithful float64 oracle, pixel by pixel.

Frames (clamped, as the node returns them) and the full-resolution flow / mask planes of the last pass (debug_state,
x64-padded) against the oracle's clamped frame and its flow{last} / mask{last}, for both operand types.  Each case's
bound is MARGIN (4) x the maximum the host emulation of the same case showed (tests/rife16_util.py, OBSERVED); it holds
over the whole plane and over the border band (2 rows / columns along every edge of the image and of the padded plane),
and a failure names the worst pixel.  The oracle runs in float64 on the same device.
"""
import pytest
import torch

import rife16_util as U

pytestmark = pytest.mark.gpu
OPERANDS = ["float16", "bfloat16"]


def _check(label, arch, sd, fr, f0, f1, ts, sf, operand, batch=8, compare_tasks=None):
    from cfi_b200.engine import Rife46Engine
    eng = Rife46Engine(sd, 0, operand, batch=batch)
    try:
        frd = fr.cuda().contiguous()
        out = eng.forward(frd, f0, f1, ts, scale_factor=sf)
        flow, mask = eng.debug_state(len(ts))
        torch.cuda.synchronize()
    finally:
        eng.close()
    sel = list(range(len(ts))) if compare_tasks is None else list(compare_tasks)
    sdd = {k: v.cuda() for k, v in sd.items()}
    want = U.oracle(arch, sdd, frd, [f0[i] for i in sel], [f1[i] for i in sel], [ts[i] for i in sel], sf, operand,
                    device="cuda")
    got = (out[sel], flow[sel], mask[sel])
    lines, fails = U.compare(f"{label} {operand}", got, want, fr.shape[1], fr.shape[2], U.tol(label, operand))
    print("\n".join(lines))
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("operand", OPERANDS)
@pytest.mark.parametrize("arch,sf,h,w", [pytest.param(*c, id=U.case_id(*c)) for c in U.cases()])
def test_rife_whole_path_matches_faithful_oracle(pkg, arch, sf, h, w, operand):
    sd, fr = U.inputs(arch, h, w)
    n = len(U.TIMESTEPS)
    _check(U.case_id(arch, sf, h, w), arch, sd, fr, [0] * n, [1] * n, list(U.TIMESTEPS), sf, operand)


@pytest.mark.parametrize("operand", OPERANDS)
def test_rife_1080p_batch8_matches_faithful_oracle(pkg, operand):
    """1080x1920 (padded to 1088 rows), batch 8 over three frames; the oracle for the first and the last task.  No host
    calibration exists at this size: the bound is MARGIN x the largest error of any calibrated case."""
    sd = U.O.synthetic_state_dict(U.SEEDS["4.6"], U.GAIN)
    fr = U.O.synthetic_clip(3, 1080, 1920, seed=1080)
    f0, f1 = [0, 0, 0, 0, 1, 1, 1, 1], [1, 1, 1, 1, 2, 2, 2, 2]
    ts = [0.05, 0.3, 0.5, 0.7, 0.2, 0.5, 0.8, 0.95]
    _check("4.6-1080x1920", "4.6", sd, fr, f0, f1, ts, 1.0, operand, batch=8, compare_tasks=(0, 7))
