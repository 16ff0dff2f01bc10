"""-m gpu: the streamed-weight tapconv mode (the ResConvs of blocks 0-2, c = 192 / 128 / 96: the whole window of a tile
staged once, the weights streamed through shared-memory slots shared by both MMA warpgroups, n_cta = 96 / 128 / 96).

Every streamed layer in fp16 and bf16 against the float64 operator on the same 16-bit inputs and packed weights, and
against the CUDA-core checker (impl=1), with the per-element bound of test_gpu_layers.py.  Outputs go into the slice
[1:B+1] of a NaN-filled buffer of B + 2 images, so a store outside the output or a cell left unwritten shows.  Partial
tiles in both directions, odd tile counts per CTA (the second warpgroup sits out the last pass) and the 1080p batch-8
geometry, where every CTA walks several passes and the weight ring and window stages wrap many times.
"""
import pytest
import torch

from gpu_util import rel_err
from oracle import rife46 as O
from test_gpu_layers import _assert_bound, _resconv_ref, _tdt

pytestmark = pytest.mark.gpu

BLOCK_C = (192, 128, 96, 64, 32)
WSTREAM_BLOCKS = (0, 1, 2)
RESCONV_LAYERS = list(range(2, 10))
# (n_cta, nsplit) of the streamed plan: all channels per CTA up to the wgmma's N = 128, else two halves
EXPECT_SPLIT = {192: (96, 2), 128: (128, 1), 96: (96, 1)}


@pytest.fixture(scope="module")
def engines(pkg):
    from cfi_b200.engine import Rife46Engine
    sd = O.synthetic_state_dict(23)
    e = {"float16": Rife46Engine(sd, 0, "float16"), "bfloat16": Rife46Engine(sd, 0, "bfloat16")}
    yield sd, e
    for v in e.values():
        v.close()


def _check_plan(eng, nblocks):
    for b in range(nblocks):
        for l in range(11):
            pl = eng.layer_plan(b, l)
            want = b in WSTREAM_BLOCKS and l in RESCONV_LAYERS
            assert pl["wstream"] == want, (b, l, pl)
            if want:
                assert (pl["n_cta"], pl["nsplit"]) == EXPECT_SPLIT[BLOCK_C[b]], (b, l, pl)
                assert not pl["cmajor"] and pl["stages"] >= 2 and pl["smem_bytes"] <= 232448, (b, l, pl)


def test_plan_selects_wide_resconvs(engines):
    """Exactly the eight ResConvs of blocks 0, 1 and 2 stream their weights."""
    _, e = engines
    for eng in e.values():
        _check_plan(eng, 4)


def test_plan_selects_wide_resconvs_arch426(pkg):
    from cfi_b200.engine import Rife46Engine
    eng = Rife46Engine(O.synthetic_state_dict(17, arch="4.26"), 0, "float16", arch="4.26")
    try:
        _check_plan(eng, 5)
    finally:
        eng.close()


def _guarded(shape, dtype):
    buf = torch.full((shape[0] + 2,) + tuple(shape[1:]), float("nan"), dtype=dtype, device="cuda")
    return buf, buf[1:shape[0] + 1]


def _sentinels_intact(buf):
    return bool(torch.isnan(buf[0].float()).all() and torch.isnan(buf[-1].float()).all())


def _run(eng, block, layer, x, impl):
    buf, out = _guarded(x.shape, x.dtype)
    eng.debug_layer(block, layer, x, out, impl=impl)
    torch.cuda.synchronize()
    assert _sentinels_intact(buf), f"block {block} layer {layer} impl {impl}: store outside the output"
    assert not torch.isnan(out.float()).any(), f"block {block} layer {layer} impl {impl}: cell left unwritten"
    return out


SHAPES = [pytest.param((3, 21, 29), id="3x21x29"), pytest.param((2, 19, 5), id="2x19x5"),
          pytest.param((1, 40, 24), id="1x40x24")]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
@pytest.mark.parametrize("layer", RESCONV_LAYERS)
@pytest.mark.parametrize("block", WSTREAM_BLOCKS)
def test_wstream_layer(engines, block, layer, dtype, shape):
    sd, e = engines
    eng, c, tdt = e[dtype], BLOCK_C[block], _tdt(dtype)
    g = torch.Generator().manual_seed(1000 * block + 10 * layer + len(shape))
    x = (0.5 * torch.randn(*shape, c, generator=g)).to(tdt)
    out = _run(eng, block, layer, x.cuda(), 0).cpu()
    chk = _run(eng, block, layer, x.cuda(), 1).cpu()
    ref, S = _resconv_ref(sd, f"block{block}.convblock.{layer - 2}.", x, dtype)
    label = f"block {block} ResConv {layer - 2} {dtype} {tuple(shape)}"
    _assert_bound(label, out, ref, S, 9 * c, tdt)
    _assert_bound(label + " (checker)", chk, ref, S, 9 * c, tdt)


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
@pytest.mark.parametrize("block", WSTREAM_BLOCKS)
def test_wstream_1080p_batch8(engines, block, dtype):
    """The 1080p geometry at batch 8 (34 x 60, 68 x 120, 136 x 240 cells): several passes per CTA, passes with two
    tiles and with one."""
    _, e = engines
    eng, c = e[dtype], BLOCK_C[block]
    s = 8 >> block
    g = torch.Generator().manual_seed(500 + block)
    x = (0.5 * torch.randn(8, 1088 // (4 * s), 1920 // (4 * s), c, generator=g)).to(_tdt(dtype)).cuda()
    out = _run(eng, block, 5, x, 0)
    chk = _run(eng, block, 5, x, 1)
    assert rel_err(out.float(), chk.float()) < (4e-3 if dtype == "float16" else 2e-2)
