"""-m gpu: conv0.0 -> conv0.1 of RIFE 4.6's 64-channel block as one launch (conv0_fused_kernel, csrc/tapconv.cu) against
the two launches it replaces (conv0.0 into the space-to-depth c00 map, conv0.1 from it).

The fused kernel issues the same products in the same K order into fp32 and rounds conv0.0's output to 16 bits where
the two launches store it, so its output must be bit-identical to theirs, not merely close.  Shapes: frames where every
tile touches the image edge (the zero c00 border and the TMA zero-fill), grids with odd numbers of tile rows and columns,
a grid with partial tiles, and 1080p at batch 8; then a whole 63-pair forward call, fused against unfused.
"""
import pytest
import torch

from oracle import rife46 as O

pytestmark = pytest.mark.gpu

LIMIT = 232448  # shared memory per CTA on sm_90 (227 KB)


@pytest.fixture(scope="module")
def engines(pkg):
    from cfi_b200.engine import Rife46Engine
    sd = O.synthetic_state_dict(5)
    e = {"float16": Rife46Engine(sd, 0, "float16"), "bfloat16": Rife46Engine(sd, 0, "bfloat16")}
    yield e
    for v in e.values():
        v.close()


def _tdt(dtype):
    return torch.float16 if dtype == "float16" else torch.bfloat16


def test_plan(engines):
    """Block 3 (c = 64) fuses, with two x window stages, within shared memory and without spills; blocks 0-2 do not."""
    for eng in engines.values():
        for b in range(3):
            assert not eng.conv0_plan(b)["fused"], b
        pl = eng.conv0_plan(3)
        print("fused conv0 plan:", pl)
        assert pl["fused"] and pl["stages"] == 2, pl
        assert 0 < pl["smem_bytes"] <= LIMIT and 0 < pl["regs"] <= 224 and pl["local_bytes"] == 0, pl


def test_other_archs_do_not_fuse(pkg):
    """Arch 4.7's block inputs hold 128 channels per cell: no block of it runs fused."""
    from cfi_b200.engine import Rife46Engine
    eng = Rife46Engine(O.synthetic_state_dict(5, arch="4.7"), 0, "float16")
    try:
        for b in range(4):
            assert not eng.conv0_plan(b)["fused"], b
    finally:
        eng.close()


# (B, H, W) of the block input x (conv0.0's grid; the output is H/2 x W/2, in tiles of 8 x 8)
SHAPES = [
    (2, 32, 32),     # 64 x 64 frames: 2 x 2 tiles, every one on the edge
    (2, 32, 64),     # 64 x 128 frames
    (3, 64, 96),     # 96 x 160 frames (padded to 128 x 192)
    (2, 48, 80),     # 3 x 5 tiles: odd numbers of tile rows and columns
    (2, 44, 52),     # partial tiles in both directions
    (8, 544, 960),   # 1080p (padded to 1088 x 1920) at batch 8
]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_fused_equals_two_launches(engines, dtype, shape):
    eng = engines[dtype]
    b, h, w = shape
    g = torch.Generator().manual_seed(h * 1000 + w)
    x = (0.5 * torch.randn(b, h, w, 64, generator=g)).to(_tdt(dtype)).cuda()
    c00 = torch.empty(b, h // 2, w // 2, 128, dtype=x.dtype, device="cuda")
    eng.debug_layer(3, 0, x, c00)
    ref = torch.empty(b, h // 2, w // 2, 64, dtype=x.dtype, device="cuda")
    eng.debug_layer(3, 1, c00, ref)
    # guard images on both sides: the fused launch writes exactly its B images
    buf = torch.full((b + 2, h // 2, w // 2, 64), float("nan"), dtype=x.dtype, device="cuda")
    eng.debug_conv0_fused(3, x, buf[1:b + 1])
    torch.cuda.synchronize()
    assert torch.isnan(buf[0].float()).all() and torch.isnan(buf[-1].float()).all()
    out = buf[1:b + 1]
    assert torch.equal(out, ref), (out.float() - ref.float()).abs().max().item()


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_forward_fused_equals_unfused(engines, dtype):
    """A whole 1080p forward call of 63 pairs: the frames are identical with block 3's conv0 pair fused or as two
    launches."""
    eng = engines[dtype]
    frames = O.synthetic_clip(64, 1080, 1920, seed=31).cuda()
    f0, f1, ts = list(range(63)), list(range(1, 64)), [0.5] * 63
    try:
        eng.set_unfused_conv0(True)
        ref = eng.forward(frames, f0, f1, ts).clone()
        eng.set_unfused_conv0(False)
        out = eng.forward(frames, f0, f1, ts)
        torch.cuda.synchronize()
    finally:
        eng.set_unfused_conv0(False)
    assert torch.equal(out, ref), (out - ref).abs().max().item()
