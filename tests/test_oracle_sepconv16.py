"""The 16-bit-faithful mode of oracle/sepconv.py (``operand=``) and the head gain of its synthetic weights, on the CPU.

Without an operand the oracle is the fp32 graph that tests/test_oracle_sepconv.py pins to the reference's outputs, and
the head gain's default must leave the synthetic weights as they were: neither may change one bit.  With an operand the
graph runs in float64 and every tensor the library stores in 16 bits is exactly representable in that type.  The
whole-path cases of tests/sepconv16_util.py must make the trunk visible in the coefficients and keep every normaliser far
from the 0.01 threshold.
"""
import os
import sys

import pytest
import torch

import sepconv16_util as U
from oracle import sepconv as OS
from oracle.rife46 import q16

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden_sepconv import sepconv_cases, sepconv_inputs  # noqa: E402

NAMES = ["sepconv_net_21x30", "sepconv_net_45x54", "sepconv_net_48x64"]


def _run(name, taps, **kw):
    cfg = sepconv_cases()[name]
    sd = OS.synthetic_state_dict(cfg["seed"])
    x = sepconv_inputs(cfg).permute(0, 3, 1, 2).contiguous()
    return OS.network_forward(sd, x[0:1], x[1:2], taps, **kw)


def _flat(v):
    return [v] if isinstance(v, torch.Tensor) else [t for x in v for t in _flat(x)]


@pytest.mark.parametrize("name", NAMES)
def test_no_operand_is_the_fp32_graph_bit_for_bit(name):
    a, b = {}, {}
    out = _run(name, a, operand=None)
    ref = _run(name, b)                                        # no operand argument at all
    assert out.dtype == torch.float32 and torch.equal(out, ref)
    assert a.keys() == b.keys() and "stats" not in a
    for k in a:
        assert all(x.dtype == torch.float32 and torch.equal(x, y) for x, y in zip(_flat(a[k]), _flat(b[k]))), k
    seed = sepconv_cases()[name]["seed"]
    s1, s2 = OS.synthetic_state_dict(seed), OS.synthetic_state_dict(seed, 1.0)
    assert all(torch.equal(s1[k], s2[k]) for k in s1)


@pytest.mark.parametrize("operand", ["float16", "bfloat16"])
@pytest.mark.parametrize("name", NAMES)
def test_operand_rounds_where_the_library_stores_16_bits(name, operand):
    dt = torch.float16 if operand == "float16" else torch.bfloat16
    taps = {}
    out = _run(name, taps, operand=operand)
    assert out.dtype == torch.float64
    assert len(taps["levels"]) == 5
    for r, t in enumerate(taps["levels"]):                     # row 0 (netInput + PReLU) and the decoded rows 1..4
        assert t.dtype == torch.float64 and torch.equal(q16(t, dt), t), r
    for k in U.PLANES:                                         # the heads' 51 coefficients
        assert taps[k].dtype == torch.float64 and torch.equal(q16(taps[k], dt), taps[k]), k
    assert taps["mean"].dtype == torch.float64 and torch.equal(taps["mean"].float().double(), taps["mean"])
    assert taps["stats"].shape == (1, 2) and taps["stats"].dtype == torch.float64
    # and it is still the same model: tens of dB of agreement with the fp32 graph
    mse = float(((out - _run(name, None).double()) ** 2).mean())
    assert mse < 10 ** -6.0, mse


@pytest.mark.parametrize("case", [pytest.param(c, id=c[0]) for c in U.PATH_CASES])
def test_path_cases_show_the_trunk_and_keep_the_normaliser_large(case):
    """On TRUNK_CASES (head gain TRUNK_GAIN), max |coef - bias| >= TRUNK_SHARE x max |bias| on every plane; on every case
    the normaliser is >= MIN_NORM at every pixel."""
    sd, fr = U.path_inputs(case)
    x = fr[..., :3].permute(0, 3, 1, 2)
    taps = {}
    OS.network_forward(sd, x[0:1], x[1:2], taps, operand="float16")
    if case[0] in U.TRUNK_CASES:
        assert case[4] == U.TRUNK_GAIN
        for k, head in zip(U.PLANES, U.HEADS):
            bias = sd[head + ".netMain.3.bias"].double().view(1, -1, 1, 1)
            share = float((taps[k] - bias).abs().max() / bias.abs().max())
            assert share >= U.TRUNK_SHARE, (k, share)
    n = OS.op64(OS.pad_frames(x[0:1]), taps["ver1"], taps["hor1"])[:, 3] + \
        OS.op64(OS.pad_frames(x[1:2]), taps["ver2"], taps["hor2"])[:, 3]
    assert float(n.abs().min()) >= U.MIN_NORM, float(n.abs().min())
