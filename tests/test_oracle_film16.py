"""The 16-bit-faithful mode of oracle/film.py (``operand=``) on the CPU.

Without an operand the oracle is the fp32 graph that tests/test_oracle_film.py pins to the reference's outputs: the hook
must not change one bit of it.  With an operand it runs in float64 and every tensor the library stores in 16 bits is
exactly representable in that type, while the flows are not even fp32-rounded.
"""
import os
import sys

import pytest
import torch

from oracle import film as OF
from oracle.rife46 import q16

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden_film import film_cases, film_inputs  # noqa: E402

NAMES = ["film_net_64x64_rand", "film_net_72x104", "film_net_128x192"]


def _run(name, taps, **kw):
    cfg = film_cases()[name]
    sd = OF.synthetic_state_dict(cfg["seed"], cfg["flow_gain"])
    x = film_inputs(cfg).permute(0, 3, 1, 2)
    return OF.interpolator_forward(sd, x[0:1], x[1:2], torch.full((1, 1), 0.5), taps, **kw)


def _flat(v):
    return [v] if isinstance(v, torch.Tensor) else [t for x in v for t in _flat(x)]


@pytest.mark.parametrize("name", NAMES)
def test_no_operand_is_the_fp32_graph_bit_for_bit(name):
    a, b = {}, {}
    out = _run(name, a, operand=None)
    ref = _run(name, b)                                        # no operand argument at all
    assert out.dtype == torch.float32 and torch.equal(out, ref)
    assert a.keys() == b.keys()
    for k in a:
        assert all(x.dtype == torch.float32 and torch.equal(x, y) for x, y in zip(_flat(a[k]), _flat(b[k]))), k
    x = torch.randn(3, 5)
    assert q16(x, None) is x


@pytest.mark.parametrize("operand", ["float16", "bfloat16"])
@pytest.mark.parametrize("name", NAMES)
def test_operand_rounds_where_the_library_stores_16_bits(name, operand):
    dt = torch.float16 if operand == "float16" else torch.bfloat16
    taps = {}
    out = _run(name, taps, operand=operand)
    assert out.dtype == torch.float64
    for frame in taps["feature_pyramids"]:                     # every feature level: T
        for l, f in enumerate(frame):
            assert f.dtype == torch.float64 and torch.equal(f.to(dt).double(), f), l
    for l, a in enumerate(taps["aligned"]):                    # warped images, features and 0.5-scaled flows: T
        assert a.dtype == torch.float64 and torch.equal(a.to(dt).double(), a), l
    for k in ("forward_flow_levels", "backward_flow_levels"):
        assert len(taps[k]) == OF.PYRAMID_LEVELS
        v = taps[k][0]                                         # flows: float64, not even fp32-rounded
        assert v.dtype == torch.float64 and not torch.equal(v.float().double(), v)
        assert all(torch.equal(a, b) for a, b in zip(taps[k][:OF.FUSION_PYRAMID_LEVELS],
                                                     taps[k.replace("_levels", "")]))
    # and it is still the same model: tens of dB of agreement with the fp32 graph
    mse = float(((out - _run(name, None).double()) ** 2).mean())
    assert mse < 10 ** -4.0, mse                               # > 40 dB (bf16: 45-47 dB, fp16: 64-65 dB)
