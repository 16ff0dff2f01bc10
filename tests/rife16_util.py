"""The whole RIFE path against the 16-bit-faithful float64 oracle (oracle/rife46.py, ``operand=``), pixel by pixel.

Shared by tests/test_rife_full_host.py (the library's schedule and CUDA-core checker compiled for the host) and
tests/test_gpu_rife16.py (the wgmma path on the GPU).  A whole-frame PSNR dilutes an error confined to one column or a
border; a max-abs bound over every pixel, and again over a band of 2 rows / columns along every edge of the image and
of the x64-padded plane, does not, and the worst pixel's location is reported.

There is no a-priori bound for the whole path: fp32 accumulation order flips a 16-bit store by one ulp now and then and
the flip propagates through the later layers and the warps, most where a warp samples across the edge between the image
and its zero padding.  So each case's bound is MARGIN x the error the host emulation showed on that case (OBSERVED).
How large that propagation is shows in the oracle itself: evaluated with fp32 instead of float64 accumulation it moves by
the same order (fp16: 1.8e-4 in the frame, 4e-3 px of flow on ifnet_64x64_gain4).
"""
from typing import Dict, List, Tuple

import torch

from oracle import rife46 as O

MARGIN = 4.0
# max |engine - oracle| (frame, flow in px, mask) of the host emulation, per case and operand type; the matrix cases
# (case_id) first, then the golden cases of test_rife_full_host.py
OBSERVED = {  # case: (float16 (frame, flow, mask), bfloat16 (frame, flow, mask))
    "4.6-sf1-97x131": ((9.02e-03, 1.79e-02, 9.07e-03), (3.58e-02, 8.78e-02, 6.27e-02)),
    "4.6-sf1-200x72": ((6.92e-03, 1.36e-02, 7.68e-03), (4.57e-02, 1.02e-01, 5.56e-02)),
    "4.6-sf1-7x200": ((2.74e-03, 9.09e-03, 4.45e-03), (1.37e-02, 4.59e-02, 3.52e-02)),
    "4.7-sf1-97x131": ((3.04e-03, 1.01e-02, 5.68e-03), (3.34e-02, 8.66e-02, 4.36e-02)),
    "4.7-sf1-200x72": ((3.48e-03, 1.01e-02, 5.39e-03), (1.95e-02, 8.05e-02, 4.60e-02)),
    "4.7-sf1-7x200": ((1.60e-03, 5.84e-03, 3.86e-03), (1.03e-02, 3.34e-02, 2.23e-02)),
    "4.17-sf1-97x131": ((4.40e-03, 1.01e-02, 4.82e-03), (2.10e-02, 7.21e-02, 3.79e-02)),
    "4.17-sf1-200x72": ((4.69e-03, 1.15e-02, 4.56e-03), (5.04e-02, 8.68e-02, 3.33e-02)),
    "4.17-sf1-7x200": ((1.45e-03, 5.00e-03, 2.94e-03), (6.04e-03, 4.99e-02, 2.74e-02)),
    "4.26-sf1-97x131": ((2.42e-03, 6.49e-03, 1.76e-03), (1.01e-02, 5.26e-02, 1.30e-02)),
    "4.26-sf1-200x72": ((3.01e-03, 8.51e-03, 2.00e-03), (1.84e-02, 5.85e-02, 2.26e-02)),
    "4.26-sf1-7x200": ((7.71e-04, 3.71e-03, 1.12e-03), (5.77e-03, 2.54e-02, 8.24e-03)),
    "4.6-sf0.25-100x203": ((6.09e-03, 1.71e-02, 2.63e-03), (4.36e-02, 1.21e-01, 1.93e-02)),
    "4.6-sf0.5-100x203": ((6.66e-03, 2.33e-02, 4.49e-03), (3.11e-02, 1.03e-01, 3.85e-02)),
    "4.6-sf2-37x101": ((2.94e-03, 7.24e-03, 5.98e-03), (2.09e-02, 4.72e-02, 4.29e-02)),
    "4.6-sf4-37x101": ((1.42e-03, 3.87e-03, 4.45e-03), (8.71e-03, 2.84e-02, 3.53e-02)),
    "4.26-sf0.25-203x230": ((2.17e-03, 1.19e-02, 6.51e-04), (3.35e-02, 8.59e-02, 5.21e-03)),
    "4.26-sf0.5-100x203": ((2.66e-03, 8.11e-03, 7.26e-04), (1.32e-02, 6.27e-02, 4.86e-03)),
    "4.26-sf2-37x101": ((9.98e-04, 3.58e-03, 9.46e-04), (8.81e-03, 2.58e-02, 8.47e-03)),
    "4.26-sf4-37x101": ((6.98e-04, 3.04e-03, 1.08e-03), (7.81e-03, 2.47e-02, 8.88e-03)),
    "ifnet_64x64_gain4": ((2.22e-04, 7.19e-03, 4.03e-03), (1.54e-03, 3.22e-02, 2.38e-02)),
    "ifnet47_64x128_gain3": ((1.94e-04, 4.59e-03, 2.10e-03), (1.26e-03, 2.33e-02, 1.50e-02)),
    "ifnet417_64x128_gain3": ((1.60e-04, 3.31e-03, 1.67e-03), (1.10e-03, 3.35e-02, 1.01e-02)),
    "ifnet426_128x128_gain3": ((1.85e-04, 4.61e-03, 1.25e-03), (1.33e-03, 1.53e-02, 9.32e-03)),
    "ifnet_64x64_sf2": ((7.30e-05, 1.96e-03, 1.31e-03), (5.96e-04, 1.62e-02, 1.02e-02)),
    "ifnet_64x64_sf4": ((5.24e-05, 1.43e-03, 1.52e-03), (4.37e-04, 1.08e-02, 1.22e-02)),
    "ifnet47_64x64_sf2": ((6.24e-05, 1.53e-03, 3.72e-04), (3.84e-04, 1.07e-02, 3.37e-03)),
    "ifnet47_64x64_sf4": ((3.61e-05, 9.71e-04, 5.27e-04), (2.50e-04, 7.81e-03, 4.23e-03)),
    "ifnet417_64x64_sf2": ((5.13e-05, 1.52e-03, 3.95e-04), (4.03e-04, 1.23e-02, 2.48e-03)),
    "ifnet426_64x64_sf2": ((3.69e-05, 1.16e-03, 1.76e-04), (2.16e-04, 6.46e-03, 1.46e-03)),
    "ifnet426_64x64_sf4": ((3.71e-05, 9.23e-04, 2.46e-04), (2.76e-04, 7.77e-03, 2.63e-03)),
    "ifnet_40x100_sf2": ((9.71e-04, 2.56e-03, 1.57e-03), (4.40e-03, 1.94e-02, 1.22e-02)),
    "ifnet426_40x100_sf4": ((3.04e-04, 1.55e-03, 4.02e-04), (1.67e-03, 6.36e-03, 2.48e-03)),
}


def tol(case: str, operand: str) -> Dict[str, float]:
    """MARGIN x what the host emulation showed for this case; a case it cannot run (1080p) gets the largest over all."""
    i = 0 if operand == "float16" else 1
    obs = OBSERVED[case][i] if case in OBSERVED else tuple(max(v[i][k] for v in OBSERVED.values()) for k in range(3))
    return dict(zip(("frame", "flow", "mask"), (MARGIN * v for v in obs)))


ARCHS = ("4.6", "4.7", "4.17", "4.26")
SIZES = ((97, 131), (200, 72), (7, 200))       # neither dimension a multiple of 8, and a thin strip
TIMESTEPS = (0.05, 0.5, 0.95)
GAIN = 4.0                                      # lastconv x4: flows of several pixels, warps that reach the border
SEEDS = {"4.6": 101, "4.7": 102, "4.17": 103, "4.26": 104}
# node scale_factor: block scales / scale_factor (0.25, 0.5: coarser blocks; 2, 4: the last blocks up-scaled)
# (sizes whose padded plane divides by every block scale, as the reference needs; 4.26 at 0.25 runs a scale-64 block)
SCALE_CASES = (("4.6", 0.25, 100, 203), ("4.6", 0.5, 100, 203), ("4.6", 2.0, 37, 101), ("4.6", 4.0, 37, 101),
               ("4.26", 0.25, 203, 230), ("4.26", 0.5, 100, 203), ("4.26", 2.0, 37, 101), ("4.26", 4.0, 37, 101))


def cases() -> List[Tuple[str, float, int, int]]:
    """(arch, scale_factor, h, w) of the whole-path matrix."""
    return [(a, 1.0, h, w) for a in ARCHS for h, w in SIZES] + list(SCALE_CASES)


def case_id(arch, sf, h, w):
    return f"{arch}-sf{sf:g}-{h}x{w}"


def inputs(arch: str, h: int, w: int):
    """(state dict, frames [2,h,w,3] fp32 NHWC) of one case."""
    sd = O.synthetic_state_dict(SEEDS[arch], GAIN, arch=arch)
    fr = O.synthetic_clip(2, h, w, seed=SEEDS[arch] + 1000 * h + w)
    return sd, fr


def oracle(arch: str, sd, fr: torch.Tensor, f0, f1, ts, sf: float, operand: str, device="cpu"):
    """The faithful oracle's (frame [B,h,w,3] clamped, flow [B,Hp,Wp,4], mask [B,Hp,Wp]) for tasks (f0[i], f1[i], ts[i])."""
    x = fr.to(device).permute(0, 3, 1, 2)
    taps: Dict[str, torch.Tensor] = {}
    sl = [v / sf for v in O.SCALE_LIST[arch]]
    t = torch.tensor(list(ts), dtype=torch.float32).view(-1, 1, 1, 1)
    out = O.ifnet_forward(arch, sd, x[list(f0)], x[list(f1)], t, sl, taps, operand)
    last = len(sl) - 1
    return (out.clamp(0, 1).permute(0, 2, 3, 1), taps[f"flow{last}"].permute(0, 2, 3, 1), taps[f"mask{last}"][:, 0])


def border_band(H: int, W: int, h: int, w: int, device="cpu") -> torch.Tensor:
    """[H, W] bool: the first and last 2 rows and columns of the h x w image and of the H x W plane it sits in."""
    rows = torch.zeros(H, dtype=torch.bool, device=device)
    cols = torch.zeros(W, dtype=torch.bool, device=device)
    for n, v in ((h, rows), (H, rows)):
        v[:2] = True
        v[max(n - 2, 0):n] = True
    for n, v in ((w, cols), (W, cols)):
        v[:2] = True
        v[max(n - 2, 0):n] = True
    return rows[:, None] | cols[None, :]


def _worst(err: torch.Tensor, sel: torch.Tensor = None):
    """(max |err|, its index (b, y, x[, c])) over err [B, H, W(, C)], optionally restricted to pixels sel [H, W]."""
    e = err if sel is None else torch.where(sel.view(1, *sel.shape, *([1] * (err.dim() - 3))), err, torch.zeros_like(err))
    i = int(torch.argmax(e))
    idx = []
    for d in reversed(e.shape):
        idx.append(i % d)
        i //= d
    return float(e.max()), tuple(reversed(idx))


def compare(label: str, got, want, h: int, w: int, tol: Dict[str, float], names=("frame", "flow", "mask")):
    """Max-abs comparison of the planes ``names`` (default: frame, flow, mask) over everything and over the border band;
    returns the report lines and the list of failures (empty when every bound holds)."""
    lines, fails = [], []
    for name, g, r in zip(names, got, want):
        err = (g.to(r.device).double() - r.double()).abs()
        H, W = err.shape[1], err.shape[2]
        band = border_band(H, W, h, w, err.device)
        for where, sel in (("all", None), ("border", band)):
            v, at = _worst(err, sel)
            ratio = v / tol[name]
            lines.append(f"{label} {name:5s} {where:6s}: max |err| {v:.3e} at (b,y,x[,c]) {at}, {ratio:.2f} of the bound")
            if not v <= tol[name]:
                fails.append(lines[-1])
    return lines, fails
