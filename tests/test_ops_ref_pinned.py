"""Pin oracle/ops_ref.py (the CPU restatements the sm_90a op kernels are checked against on the GPU) to the REFERENCE'S OWN
kernels: the cupy kernel strings of vfi_models/ops/cupy_ops, specialised by the reference's own pre-processor and executed
on the CPU through tests/host_emu (oracle/ref_ops.py).  Their outputs on these seeded inputs are stored, with the inputs, in
tests/golden/ref_ops_kernels.npz (tools/make_golden_ref_ops.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import ops_ref

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_ops_kernels.npz"))


def _case(name):
    return {k.split("/", 1)[1]: torch.from_numpy(GOLD[k]) for k in GOLD.files if k.startswith(name + "/")}


@pytest.mark.parametrize("shape,mag", [((1, 3, 9, 13), 1.5), ((2, 5, 8, 8), 6.0)])
def test_softsplat_sum_matches_reference_kernel(shape, mag):
    d = _case(f"splat_{shape[1]}")
    assert tuple(d["x"].shape) == shape and float(d["flow"].abs().max()) <= mag   # some targets fall outside
    got = ops_ref.softsplat_sum(d["x"], d["flow"])
    assert (got - d["ref"]).abs().max().item() <= 1e-5


def test_softsplat_modes_on_top_of_the_reference_kernel():
    """softsplat() (cupy_ops/softsplat.py:382-435) = host arithmetic around softsplat_out; with the kernel being the
    reference's, 'avg' and 'soft' of the oracle must agree with that arithmetic done here."""
    d = _case("modes_avg")
    x, flow, metric = d["x"], d["flow"], d["metric"]
    o = d["ref"]
    norm = o[:, -1:].clone()
    norm[norm == 0.0] = 1.0
    assert (ops_ref.softsplat(x, flow, None, "avg") - o[:, :-1] / norm).abs().max().item() <= 2e-4  # small normalisers amplify fp32 rounding
    o = _case("modes_soft")["ref"]
    norm = o[:, -1:].clone()
    norm[norm == 0.0] = 1.0
    assert (ops_ref.softsplat(x, flow, metric, "soft") - o[:, :-1] / norm).abs().max().item() <= 2e-4  # small normalisers amplify fp32 rounding


@pytest.mark.parametrize("shape", [(1, 8, 6, 7), (2, 3, 10, 5)])
def test_costvol_matches_reference_kernel(shape):
    d = _case(f"costvol_{shape[2]}")
    assert tuple(d["one"].shape) == shape
    assert (ops_ref.costvol_l1(d["one"], d["two"]) - d["ref"]).abs().max().item() <= 1e-5


@pytest.mark.parametrize("k,hw", [(5, (6, 7)), (51, (4, 3))])
def test_sepconv_matches_reference_kernel(k, hw):
    d = _case(f"sepconv_{k}")
    assert tuple(d["ver"].shape) == (1, k, *hw)
    ref = d["ref"]
    got = ops_ref.sepconv(d["x"], d["ver"], d["hor"])
    assert (got - ref).abs().max().item() <= 1e-4 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("shape", [(1, 40, 5, 6), (2, 7, 4, 9)])
def test_correlation_dot_matches_reference_kernels(shape):
    """kernel_Correlation_rearrange + kernel_Correlation_updateOutput with blocks of 16 / 32 cooperating threads (fibers)."""
    d = _case(f"corr_{shape[1]}")
    assert tuple(d["a"].shape) == shape
    assert (ops_ref.correlation_dot(d["a"], d["b"]) - d["ref"]).abs().max().item() <= 1e-5


@pytest.mark.parametrize("f,dil", [(3, 1), (5, 2)])
def test_adacof_matches_reference_kernel(f, dil):
    d = _case(f"adacof_{f}")   # negative offsets in the inputs: (int) truncation != floor
    assert int(d["dil"]) == dil and d["w"].shape[1] == f * f
    ref = d["ref"]
    got = ops_ref.adacof(d["x"], d["w"], d["oi"], d["oj"], int(d["dil"]))
    assert (got - ref).abs().max().item() <= 2e-5 * max(1.0, float(ref.abs().max()))


def test_edt_matches_reference_kernel_and_scipy():
    d = _case("edt")
    data, diam2 = d["data"], float(d["diam2"])
    assert torch.equal(ops_ref.edt_pass(data, diam2), d["ref"])
    img = (data == 0).float()                                   # the feature pixels; image 1 is empty (defaults to the diameter)
    from scipy import ndimage
    want = ndimage.distance_transform_edt(1 - img[0].numpy())
    assert abs(ops_ref.batch_edt(img)[0].numpy() - want).max() <= 1e-4
    assert float(ops_ref.batch_edt(img)[1].min()) == pytest.approx(diam2 ** 0.5)
