"""-m gpu: the tapconv epilogue's output paths (TMA tensor stores from a staging tile, the ResConv residual read from the
staged window, lastconv's fp32 planes) against the CUDA-core checker (impl=1) on the same packed weights.

Guard bands: every layer writes into the slice [1:B+1] of a buffer of B + 2 images pre-filled with NaN, at shapes with
partial tiles in both directions, so a store outside the output tensor shows up as a changed sentinel.
"""
import pytest
import torch

from gpu_util import rel_err
from oracle import rife46 as O

pytestmark = pytest.mark.gpu

BLOCK_C = (192, 128, 96, 64)


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


def _tol(dtype):
    return 4e-3 if dtype == "float16" else 2e-2


def _guarded(shape, dtype):
    """(buffer of shape[0] + 2 images full of NaN, its slice [1:B+1])"""
    buf = torch.full((shape[0] + 2,) + tuple(shape[1:]), float("nan"), dtype=dtype, device="cuda")
    return buf, buf[1:shape[0] + 1]


def _sentinels_intact(buf):
    return bool(torch.isnan(buf[0].float()).all() and torch.isnan(buf[-1].float()).all())


def _run_16bit(eng, block, layer, x, cout):
    b, h, w = x.shape[:3]
    buf, out = _guarded((b, h, w, cout), x.dtype)
    eng.debug_layer(block, layer, x, out, impl=0)
    ref = torch.empty(b, h, w, cout, dtype=x.dtype, device="cuda")
    eng.debug_layer(block, layer, x, ref, impl=1)
    torch.cuda.synchronize()
    return buf, out, ref


SHAPES = [pytest.param((3, 21, 29), id="3x21x29"), pytest.param((2, 19, 5), id="2x19x5")]
DTYPES = ["float16", "bfloat16"]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("block", [3, 2, 1, 0])
def test_resconv_guard_bands(engines, block, dtype, shape):
    eng, c = engines[dtype], BLOCK_C[block]
    g = torch.Generator().manual_seed(block)
    x = (0.5 * torch.randn(*shape, c, generator=g)).to(_tdt(dtype)).cuda()
    buf, out, ref = _run_16bit(eng, block, 2 + 4, x, c)
    assert _sentinels_intact(buf)
    assert not torch.isnan(out.float()).any()
    assert rel_err(out.float(), ref.float()) < _tol(dtype)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("block", [3, 2])
def test_conv01_guard_bands(engines, block, dtype, shape):
    eng, c = engines[dtype], BLOCK_C[block]
    g = torch.Generator().manual_seed(10 + block)
    x = (0.5 * torch.randn(*shape, 2 * c, generator=g)).to(_tdt(dtype)).cuda()
    buf, out, ref = _run_16bit(eng, block, 1, x, c)
    assert _sentinels_intact(buf)
    assert not torch.isnan(out.float()).any()
    assert rel_err(out.float(), ref.float()) < _tol(dtype)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("block", [3, 2])
def test_lastconv_guard_bands(engines, block, dtype, shape):
    eng, c = engines[dtype], BLOCK_C[block]
    b, h, w = shape
    g = torch.Generator().manual_seed(20 + block)
    x = (0.5 * torch.randn(b, h, w, c, generator=g)).to(_tdt(dtype)).cuda()
    fbuf, flow = _guarded((b, 4 * h, 4 * w, 4), torch.float32)
    mbuf, mask = _guarded((b, 4 * h, 4 * w), torch.float32)
    eng.debug_layer(block, 10, x, flow, out_mask=mask, impl=0)
    rflow = torch.empty(b, 4 * h, 4 * w, 4, device="cuda")
    rmask = torch.empty(b, 4 * h, 4 * w, device="cuda")
    eng.debug_layer(block, 10, x, rflow, out_mask=rmask, impl=1)
    torch.cuda.synchronize()
    assert _sentinels_intact(fbuf) and _sentinels_intact(mbuf)
    assert not torch.isnan(flow).any() and not torch.isnan(mask).any()
    assert rel_err(flow, rflow) < 1e-4  # fp32 outputs: only accumulation order differs
    assert rel_err(mask, rmask) < 1e-4


@pytest.mark.parametrize("block,layer", [pytest.param(2, 5, id="block2-resconv"), pytest.param(2, 1, id="block2-conv01"),
                                         pytest.param(3, 1, id="block3-conv01")])
def test_many_tiles_1080p(engines, block, layer):
    """The 1080p geometry at batch 8: every persistent CTA walks many tiles, so window stages, held residual windows
    and both warpgroups' staging tiles wrap many times.  Block 2 is c = 96: a 32-channel SWIZZLE_64B tail k-block in the
    residual read and, with two output-channel splits, store boxes that start at channel n0 != 0."""
    eng, c = engines["float16"], BLOCK_C[block]
    s = (8, 4, 2, 1)[block]
    h, w = 1088 // s // 4, 1920 // s // 4
    cin = c if layer >= 2 else 2 * c
    g = torch.Generator().manual_seed(40 + block + layer)
    x = (0.5 * torch.randn(8, h, w, cin, generator=g)).half().cuda()
    buf, out, ref = _run_16bit(eng, block, layer, x, c)
    assert _sentinels_intact(buf)
    assert rel_err(out.float(), ref.float()) < _tol("float16")
