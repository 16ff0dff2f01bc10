"""The 16-bit-faithful mode of oracle/rife46.py (``operand=``) on the CPU.

Without an operand the oracle is the fp32 graph that tests/test_oracle_golden.py pins to the reference's outputs: the
hook must not change one bit of it.  With an operand it runs in float64 and every tensor the library stores or packs in
16 bits is exactly representable in that type.
"""
import os
import sys

import pytest
import torch

from oracle import rife46 as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden import cases, make_inputs  # noqa: E402

NAMES = ["ifnet_64x64_gain4", "ifnet47_64x128_gain3", "ifnet417_64x128_gain3", "ifnet426_128x128_gain3",
         "ifnet_40x100_sf2", "ifnet426_40x100_sf4"]


def _run(name, taps, **kw):
    cfg = cases()[name]
    arch = cfg.get("arch", "4.6")
    sd = O.synthetic_state_dict(cfg["seed"], cfg["gain"], arch=arch)
    x = make_inputs(cfg).permute(0, 3, 1, 2)
    ts = torch.tensor(cfg["ts"], dtype=torch.float32).view(-1, 1, 1, 1)
    sl = [v / cfg.get("scale_factor", 1.0) for v in O.SCALE_LIST[arch]]
    b = len(cfg["ts"])
    return O.ifnet_forward(arch, sd, x[0:1].repeat(b, 1, 1, 1), x[1:2].repeat(b, 1, 1, 1), ts, sl, taps, **kw)


@pytest.mark.parametrize("name", NAMES)
def test_no_operand_is_the_fp32_graph_bit_for_bit(name):
    a, b = {}, {}
    out = _run(name, a, operand=None)
    ref = _run(name, b)                                        # no operand argument at all
    assert out.dtype == torch.float32 and torch.equal(out, ref)
    assert a.keys() == b.keys() and all(v.dtype == torch.float32 and torch.equal(v, b[k]) for k, v in a.items())
    x = torch.randn(3, 5)
    assert O.q16(x, None) is x


@pytest.mark.parametrize("operand", ["float16", "bfloat16"])
@pytest.mark.parametrize("name", NAMES)
def test_operand_rounds_where_the_library_stores_16_bits(name, operand):
    dt = torch.float16 if operand == "float16" else torch.bfloat16
    taps = {}
    out = _run(name, taps, operand=operand)
    assert out.dtype == torch.float64
    blocks = [k[:-2] for k in taps if k.endswith(".x")]
    assert blocks
    for blk in blocks:
        for t in ("x", "c00", "c01", "feat"):                 # block input, conv0.0, conv0.1, ResConv outputs: T
            v = taps[f"{blk}.{t}"]
            assert v.dtype == torch.float64 and torch.equal(v.to(dt).double(), v), (blk, t)
        tmp = taps[f"{blk}.tmp"]
        if tmp.shape[1] == 13:                                 # 4.26: the fed-back features are stored in T
            assert torch.equal(tmp[:, 5:].to(dt).double(), tmp[:, 5:])
        assert not torch.equal(tmp[:, :5].to(torch.float32).double(), tmp[:, :5])  # flow / mask: not even fp32-rounded
    if "f0" in taps:                                           # encoder features: fp16 (4.7) or T (4.17, 4.26)
        fdt = torch.float16 if cases()[name].get("arch") == "4.7" else dt
        assert torch.equal(taps["f0"].to(fdt).double(), taps["f0"])
    # and it is still the same model: tens of dB of agreement with the fp32 graph
    assert O.psnr(out.float(), _run(name, None)) > 45.0
