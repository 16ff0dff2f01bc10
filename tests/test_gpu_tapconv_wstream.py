"""-m gpu: the streamed-weight tapconv mode (the whole window of a tile staged once, the weights streamed through
shared-memory slots shared by both MMA warpgroups): the ResConvs of blocks 0-2 (c = 192 / 128 / 96, n_cta = 96 / 128 /
96), block 1's lastconv (c = 128, all 80 fp32 columns in one CTA) and arch 4.26's feature conv of blocks 0 and 1
(c = 192 / 128, all 128 columns of the [B, 4H, 4W, 8] patch-form output in one CTA).

Every streamed layer in fp16 and bf16 against the float64 operator on the same 16-bit inputs and packed weights, and
against the CUDA-core checker (impl=1), with the per-element bound of test_gpu_layers.py.  Outputs go into the slice
[1:B+1] of a NaN-filled buffer of B + 2 images, so a store outside the output or a cell left unwritten shows.  Partial
tiles in both directions, odd tile counts per CTA (the second warpgroup sits out the last pass) and the 1080p batch-8
geometry, where every CTA walks several passes and the weight ring and window stages wrap many times.
"""
import pytest
import torch

from gpu_util import nhwc, rel_err
from oracle import rife46 as O
from test_gpu_layers import _assert_bound, _lastconv_ref, _resconv_ref, _tdt

pytestmark = pytest.mark.gpu

BLOCK_C = (192, 128, 96, 64, 32)
WSTREAM_BLOCKS = (0, 1, 2)
RESCONV_LAYERS = list(range(2, 10))
# (n_cta, nsplit) of the streamed ResConv plan: all channels per CTA up to the wgmma's N = 128, else two halves
EXPECT_SPLIT = {192: (96, 2), 128: (128, 1), 96: (96, 1)}


def streamed_layers(arch):
    """{(block, layer): (n_cta, nsplit)} of every layer of the arch that streams its weights."""
    want = {(b, l): EXPECT_SPLIT[BLOCK_C[b]] for b in WSTREAM_BLOCKS for l in RESCONV_LAYERS}
    want[(1, 10)] = (80, 1)  # block 1's lastconv
    if arch == "4.26":
        want[(0, 11)] = want[(1, 11)] = (128, 1)  # the feature conv at c = 192 / 128
    return want


def check_plan(plan, arch):
    """plan(block, layer) -> the layer_plan dict: exactly streamed_layers(arch) stream, with their split, and fit."""
    want = streamed_layers(arch)
    nblocks = 5 if arch == "4.26" else 4
    for b in range(nblocks):
        for l in range(12 if arch == "4.26" and b + 1 < nblocks else 11):
            pl = plan(b, l)
            assert pl["wstream"] == ((b, l) in want), (arch, b, l, pl)
            if pl["wstream"]:
                assert (pl["n_cta"], pl["nsplit"]) == want[(b, l)], (arch, b, l, pl)
                assert not pl["cmajor"] and pl["stages"] >= 2 and pl["smem_bytes"] <= 232448, (arch, b, l, pl)


def _engines(sd, arch):
    from cfi_b200.engine import Rife46Engine
    return {dt: Rife46Engine(sd, 0, dt, arch=arch) for dt in ("float16", "bfloat16")}


@pytest.fixture(scope="module")
def engines(pkg):
    sd = O.synthetic_state_dict(23)
    e = _engines(sd, "4.6")
    yield sd, e
    for v in e.values():
        v.close()


@pytest.fixture(scope="module")
def engines426(pkg):
    sd = O.synthetic_state_dict(17, arch="4.26")
    e = _engines(sd, "4.26")
    yield sd, e
    for v in e.values():
        v.close()


def test_plan_selects_streamed_layers(engines):
    """Exactly the eight ResConvs of blocks 0, 1 and 2 and block 1's lastconv stream their weights."""
    _, e = engines
    for eng in e.values():
        check_plan(eng.layer_plan, "4.6")


def test_plan_selects_streamed_layers_arch426(engines426):
    """4.26 streams the same layers and the feature conv of blocks 0 and 1."""
    _, e = engines426
    for eng in e.values():
        check_plan(eng.layer_plan, "4.26")


def _guarded(shape, dtype):
    buf = torch.full((shape[0] + 2,) + tuple(shape[1:]), float("nan"), dtype=dtype, device="cuda")
    return buf, buf[1:shape[0] + 1]


def _sentinels_intact(buf):
    return bool(torch.isnan(buf[0].float()).all() and torch.isnan(buf[-1].float()).all())


def _run(eng, block, layer, x, impl):
    """The layer's outputs on the NHWC input x: a ResConv's [B, H, W, c], lastconv's (layer 10) fp32 flow [B, 4H, 4W, 4]
    and mask [B, 4H, 4W], or the 4.26 feature conv's (layer 11) [B, 4H, 4W, 8]."""
    b, h, w = x.shape[:3]
    if layer == 10:
        guards = [_guarded((b, 4 * h, 4 * w, 4), torch.float32), _guarded((b, 4 * h, 4 * w), torch.float32)]
        eng.debug_layer(block, layer, x, guards[0][1], out_mask=guards[1][1], impl=impl)
    else:
        guards = [_guarded((b, 4 * h, 4 * w, 8) if layer == 11 else x.shape, x.dtype)]
        eng.debug_layer(block, layer, x, guards[0][1], impl=impl)
    torch.cuda.synchronize()
    for buf, out in guards:
        assert _sentinels_intact(buf), f"block {block} layer {layer} impl {impl}: store outside the output"
        assert not torch.isnan(out.float()).any(), f"block {block} layer {layer} impl {impl}: cell left unwritten"
    return [out for _, out in guards]


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
    out, = _run(eng, block, layer, x.cuda(), 0)
    chk, = _run(eng, block, layer, x.cuda(), 1)
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
    out, = _run(eng, block, 5, x, 0)
    chk, = _run(eng, block, 5, x, 1)
    assert rel_err(out.float(), chk.float()) < (4e-3 if dtype == "float16" else 2e-2)


# the streamed layers of the ConvTranspose2d + PixelShuffle lastconv: (arch, block, layer)
LAST_LAYERS = [pytest.param("4.6", 1, 10, id="block1-lastconv"), pytest.param("4.26", 0, 11, id="426-block0-features"),
               pytest.param("4.26", 1, 11, id="426-block1-features")]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
@pytest.mark.parametrize("arch,block,layer", LAST_LAYERS)
def test_wstream_lastconv(engines, engines426, arch, block, layer, dtype, shape):
    """lastconv's flow and mask planes (direct float4 / float2 stores) and the 4.26 features (patch-form direct stores)
    with streamed weights, the wgmma kernel and the checker, against the float64 operator."""
    sd, e = engines if arch == "4.6" else engines426
    eng, c, tdt = e[dtype], BLOCK_C[block], _tdt(dtype)
    g = torch.Generator().manual_seed(2000 + 100 * block + layer + len(shape))
    x = (0.5 * torch.randn(*shape, c, generator=g)).to(tdt)
    tmp, S = _lastconv_ref(sd, f"block{block}.lastconv.0.", x, dtype)
    for impl in (0, 1):
        label = f"{arch} block {block} layer {layer} {dtype} {tuple(shape)}{' (checker)' if impl else ''}"
        outs = _run(eng, block, layer, x.cuda(), impl)
        if layer == 10:
            flow, mask = outs
            _assert_bound(label + " flow", flow, nhwc(tmp[:, :4]), nhwc(S[:, :4]), 9 * c)
            _assert_bound(label + " mask", mask.unsqueeze(-1), nhwc(tmp[:, 4:5]), nhwc(S[:, 4:5]), 9 * c)
        else:
            _assert_bound(label + " features", outs[0], nhwc(tmp[:, 5:]), nhwc(S[:, 5:]), 9 * c, tdt)


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_wstream_lastconv_1080p_batch8(engines, dtype):
    """Block 1's lastconv at the 1080p geometry, batch 8 (68 x 120 cells, 600 tiles over the persistent CTAs): several
    passes per CTA, passes with two tiles and with one.  fp32 outputs: the checker differs in accumulation order only."""
    _, e = engines
    g = torch.Generator().manual_seed(600)
    x = (0.5 * torch.randn(8, 1088 // 16, 1920 // 16, 128, generator=g)).to(_tdt(dtype)).cuda()
    flow, mask = _run(e[dtype], 1, 10, x, 0)
    cflow, cmask = _run(e[dtype], 1, 10, x, 1)
    assert rel_err(flow, cflow) < 1e-4 and rel_err(mask, cmask) < 1e-4
