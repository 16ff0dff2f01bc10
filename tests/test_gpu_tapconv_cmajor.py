"""-m gpu: the channel-major tapconv MMAs (64 output channels on the wgmma M, the tile's 128 cells on N) against the
cell-major orientation of the same kernel (impl=2) and against the CUDA-core checker (impl=1).

Both orientations issue the same products in the same K order into fp32 accumulators, so their outputs are expected to
be bit-identical, not merely close.  Guard bands as in test_gpu_tapconv_epilogue.py: outputs go into the slice [1:B+1]
of a NaN-filled buffer of B + 2 images, at shapes with partial tiles in both directions.
"""
import pytest
import torch

from gpu_util import rel_err
from oracle import rife46 as O

pytestmark = pytest.mark.gpu

BLOCK_C = (192, 128, 96, 64)
# the layers that run channel-major: block 3's (c = 64) eight ResConvs.  conv0.1 (128 -> 64, 2 K=16 steps per tap)
# keeps cells on M.
CMAJOR_LAYERS = list(range(2, 10))


@pytest.fixture(scope="module")
def engines(pkg):
    from cfi_b200.engine import Rife46Engine
    sd = O.synthetic_state_dict(9)
    e = {"float16": Rife46Engine(sd, 0, "float16"), "bfloat16": Rife46Engine(sd, 0, "bfloat16")}
    yield e
    for v in e.values():
        v.close()


def _tdt(dtype):
    return torch.float16 if dtype == "float16" else torch.bfloat16


def _tol(dtype):
    return 4e-3 if dtype == "float16" else 2e-2


def _guarded(shape, dtype):
    buf = torch.full((shape[0] + 2,) + tuple(shape[1:]), float("nan"), dtype=dtype, device="cuda")
    return buf, buf[1:shape[0] + 1]


def _sentinels_intact(buf):
    return bool(torch.isnan(buf[0].float()).all() and torch.isnan(buf[-1].float()).all())


def _input(block, layer, shape, dtype, seed):
    c = BLOCK_C[block]
    g = torch.Generator().manual_seed(seed)
    return (0.5 * torch.randn(*shape, 2 * c if layer == 1 else c, generator=g)).to(_tdt(dtype)).cuda()


def _three_ways(eng, block, layer, x):
    """(guard buffer, channel-major output, cell-major output, checker output)"""
    b, h, w = x.shape[:3]
    c = BLOCK_C[block]
    buf, out = _guarded((b, h, w, c), x.dtype)
    eng.debug_layer(block, layer, x, out, impl=0)
    cell = torch.empty(b, h, w, c, dtype=x.dtype, device="cuda")
    eng.debug_layer(block, layer, x, cell, impl=2)
    ref = torch.empty(b, h, w, c, dtype=x.dtype, device="cuda")
    eng.debug_layer(block, layer, x, ref, impl=1)
    torch.cuda.synchronize()
    return buf, out, cell, ref


def _max_abs(a, b):
    return (a.float() - b.float()).abs().max().item()


def test_plan_selects_block3_conv01_and_resconvs(engines):
    """Channel-major runs exactly where the plan allows it: resident-weight 3 x 3 convs over 64 input channels with 64
    output channels per CTA and a staged 16-bit NHWC output.  For RIFE 4.6 those are block 3's ResConvs, nothing else."""
    eng = engines["float16"]
    for b in range(4):
        for l in range(11):
            pl = eng.layer_plan(b, l)
            assert pl["cmajor"] == (b == 3 and l in CMAJOR_LAYERS), (b, l, pl)
            if pl["cmajor"]:
                assert pl["n_cta"] == 64 and pl["nsplit"] == 1, (b, l, pl)


def test_plan_selects_c64_block_of_arch426(pkg):
    from cfi_b200.engine import Rife46Engine
    eng = Rife46Engine(O.synthetic_state_dict(17, arch="4.26"), 0, "float16", arch="4.26")
    try:
        for b in range(5):
            for l in range(12 if b < 4 else 11):
                assert eng.layer_plan(b, l)["cmajor"] == (b == 3 and l in CMAJOR_LAYERS), (b, l)
    finally:
        eng.close()


def test_impl_is_validated(engines):
    from cfi_b200._lib import VfiError
    eng = engines["float16"]
    x = _input(3, 2, (1, 16, 8), "float16", 0)
    with pytest.raises(VfiError):
        eng.debug_layer(3, 2, x, torch.empty_like(x), impl=3)


SHAPES = [pytest.param((3, 21, 29), id="3x21x29"), pytest.param((2, 19, 5), id="2x19x5"),
          pytest.param((1, 40, 24), id="1x40x24")]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
@pytest.mark.parametrize("layer", CMAJOR_LAYERS)
def test_cmajor_layer(engines, layer, dtype, shape):
    """Every channel-major layer: bit-identical to the cell-major MMAs, close to the checker, nothing written outside
    the output (partial border tiles are clipped by the TMA stores)."""
    eng = engines[dtype]
    x = _input(3, layer, shape, dtype, 100 + layer)
    buf, out, cell, ref = _three_ways(eng, 3, layer, x)
    assert _sentinels_intact(buf)
    assert not torch.isnan(out.float()).any()
    assert torch.equal(out, cell), f"channel-major vs cell-major: max abs diff {_max_abs(out, cell)}"
    assert rel_err(out.float(), ref.float()) < _tol(dtype)


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
@pytest.mark.parametrize("layer", [2, 9])
def test_cmajor_many_tiles_1080p(engines, layer, dtype):
    """The 1080p geometry of block 3 at batch 8 (272 x 480 cells): every persistent CTA walks many tiles, so window
    stages, held residual windows and both warpgroups' staging tiles wrap many times."""
    eng = engines[dtype]
    x = _input(3, layer, (8, 1088 // 4, 1920 // 4), dtype, 200 + layer)
    buf, out, cell, ref = _three_ways(eng, 3, layer, x)
    assert _sentinels_intact(buf)
    assert torch.equal(out, cell), f"channel-major vs cell-major: max abs diff {_max_abs(out, cell)}"
    assert rel_err(out.float(), ref.float()) < _tol(dtype)


@pytest.mark.parametrize("block,layer", [pytest.param(2, 2, id="block2-resconv"), pytest.param(3, 1, id="block3-conv01")])
def test_cell_major_switch_leaves_other_layers_alone(engines, block, layer):
    """impl=2 only changes layers the plan runs channel-major: block 2's ResConv (c = 96) and block 3's conv0.1 are the
    same launch either way."""
    eng = engines["float16"]
    x = _input(block, layer, (2, 21, 29), "float16", 300 + layer)
    a = torch.empty(*x.shape[:3], BLOCK_C[block], dtype=x.dtype, device="cuda")
    b = torch.empty_like(a)
    eng.debug_layer(block, layer, x, a, impl=0)
    eng.debug_layer(block, layer, x, b, impl=2)
    torch.cuda.synchronize()
    assert torch.equal(a, b)
