"""Write tests/golden/ref_ops_kernels.npz: the reference's own op kernels (cupy kernel strings of vfi_models/ops/cupy_ops,
run on the CPU through oracle/ref_ops.py) on the seeded inputs of tests/test_ops_ref_pinned.py, inputs and outputs both.

    VFI_REFERENCE=<reference checkout> python tools/make_golden_ref_ops.py

Needs the reference checkout and g++; the test that reads the file needs neither.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_ops  # noqa: E402


def cases():
    """(name, inputs dict, reference function of the inputs) for every case the test checks."""
    for shape, mag in (((1, 3, 9, 13), 1.5), ((2, 5, 8, 8), 6.0)):
        g = torch.Generator().manual_seed(shape[1])
        x = torch.randn(*shape, generator=g)
        flow = (torch.rand(shape[0], 2, shape[2], shape[3], generator=g) - 0.5) * 2 * mag
        yield f"splat_{shape[1]}", {"x": x, "flow": flow}, lambda d: ref_ops.softsplat_out(d["x"], d["flow"])
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1, 4, 7, 9, generator=g)
    flow = (torch.rand(1, 2, 7, 9, generator=g) - 0.5) * 5
    metric = torch.randn(1, 1, 7, 9, generator=g) * 0.3
    yield "modes_avg", {"x": x, "flow": flow, "metric": metric}, \
        lambda d: ref_ops.softsplat_out(torch.cat([d["x"], d["x"].new_ones(1, 1, 7, 9)], 1), d["flow"])
    yield "modes_soft", {"x": x, "flow": flow, "metric": metric}, \
        lambda d: ref_ops.softsplat_out(torch.cat([d["x"] * d["metric"].exp(), d["metric"].exp()], 1), d["flow"])
    for shape in ((1, 8, 6, 7), (2, 3, 10, 5)):
        g = torch.Generator().manual_seed(shape[2])
        one, two = torch.randn(*shape, generator=g), torch.randn(*shape, generator=g)
        yield f"costvol_{shape[2]}", {"one": one, "two": two}, lambda d: ref_ops.costvol_out(d["one"], d["two"])
    for k, hw in ((5, (6, 7)), (51, (4, 3))):
        g = torch.Generator().manual_seed(k)
        x = torch.randn(1, 4, hw[0] + k - 1, hw[1] + k - 1, generator=g)
        ver, hor = torch.randn(1, k, *hw, generator=g), torch.randn(1, k, *hw, generator=g)
        yield f"sepconv_{k}", {"x": x, "ver": ver, "hor": hor}, lambda d: ref_ops.sepconv_out(d["x"], d["ver"], d["hor"])
    for shape in ((1, 40, 5, 6), (2, 7, 4, 9)):
        g = torch.Generator().manual_seed(shape[1])
        a, b = torch.randn(*shape, generator=g), torch.randn(*shape, generator=g)
        yield f"corr_{shape[1]}", {"a": a, "b": b}, lambda d: ref_ops.correlation(d["a"], d["b"])
    for f, dil in ((3, 1), (5, 2)):
        g = torch.Generator().manual_seed(f)
        n, c, ho, wo = 2, 3, 6, 7
        x = torch.randn(n, c, ho + (f - 1) * dil, wo + (f - 1) * dil, generator=g)
        w = torch.randn(n, f * f, ho, wo, generator=g)
        oi = torch.randn(n, f * f, ho, wo, generator=g) * 2.5
        oj = torch.randn(n, f * f, ho, wo, generator=g) * 2.5
        yield f"adacof_{f}", {"x": x, "w": w, "oi": oi, "oj": oj, "dil": torch.tensor(dil)}, \
            lambda d: ref_ops.adacof(d["x"], d["w"], d["oi"], d["oj"], int(d["dil"]))
    g = torch.Generator().manual_seed(2)
    img = (torch.rand(2, 9, 12, generator=g) > 0.85).float()
    img[1] = 0
    diam2 = 9 ** 2 + 12 ** 2
    yield "edt", {"data": (1 - img) * diam2, "diam2": torch.tensor(float(diam2))}, \
        lambda d: ref_ops.edt_pass(d["data"], float(d["diam2"]))


def main():
    assert ref_ops.available(), "reference checkout (VFI_REFERENCE) or CUDA headers not found"
    out = {}
    for name, inputs, fn in cases():
        for k, v in inputs.items():
            out[f"{name}/{k}"] = v.numpy()
        out[f"{name}/ref"] = fn(inputs).numpy()
    path = os.path.join(ROOT, "tests", "golden", "ref_ops_kernels.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
