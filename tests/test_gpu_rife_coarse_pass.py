"""-m gpu: the wide-span schedule of vfi_rife46_forward on the H100.  The coarse blocks run over a span of many pairs per
launch, the first dense block over middle spans inside it, the other blocks in passes of `batch` pairs.  Per-pair
arithmetic does not depend on any of these widths, so a call with many tasks must give, bit for bit, the frames of one
call per task, and its debug state must be that of a call holding only its last pass's tasks.  At 1080p, 4.6 runs the
63 pairs of a 64-frame clip as one coarse span; 4.26, whose coarse part is larger, as two.  The layer plans stay those
of tests/golden/rife_layer_plans.json."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import rife46 as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (arch, scale_factor, h, w, frames, tasks, batch)
CASES = [("4.6", 1.0, 64, 64, 5, 13, 2), ("4.6", 0.5, 64, 64, 5, 13, 2), ("4.6", 2.0, 37, 60, 5, 13, 2),
         ("4.6", 4.0, 37, 60, 5, 13, 2), ("4.7", 1.0, 50, 64, 5, 13, 2), ("4.17", 1.0, 64, 50, 5, 13, 2),
         ("4.26", 1.0, 64, 64, 5, 13, 2), ("4.26", 0.5, 100, 120, 5, 13, 2), ("4.26", 2.0, 40, 64, 5, 13, 2),
         ("4.6", 1.0, 1080, 1920, 64, 63, 8), ("4.26", 1.0, 1080, 1920, 64, 63, 8)]


def _tasks(n_frames, n_tasks, seed):
    """Mixed pairs and timesteps; at 64 frames the consecutive pairs of a clip, as the node hands them over."""
    rng = np.random.default_rng(seed)
    if n_tasks == n_frames - 1:
        f0 = np.arange(n_tasks, dtype=np.int32)
    else:
        f0 = rng.integers(0, n_frames - 1, n_tasks).astype(np.int32)
    f1 = f0 + 1
    f0[3], f1[3] = f1[3], f0[3]
    return f0.tolist(), f1.tolist(), rng.uniform(0.02, 0.98, n_tasks).astype(np.float32).tolist()


@pytest.mark.parametrize("operand", ["float16", "bfloat16"])
@pytest.mark.parametrize("arch,sf,h,w,nf,nt,batch", CASES, ids=[f"{c[0]}-sf{c[1]:g}-{c[2]}x{c[3]}-{c[5]}tasks" for c in CASES])
def test_coarse_spans_match_one_call_per_task(pkg, arch, sf, h, w, nf, nt, batch, operand):
    from cfi_b200.engine import Rife46Engine
    sd = O.synthetic_state_dict(11, 3.0, arch=arch)
    fr = O.synthetic_clip(nf, h, w, seed=h + w + nt).cuda().contiguous()
    f0, f1, ts = _tasks(nf, nt, h * w)
    eng = Rife46Engine(sd, 0, operand, batch=batch, arch=arch)
    try:
        got = eng.forward(fr, f0, f1, ts, scale_factor=sf).clone()
        last = (nt - 1) // batch * batch  # the last pass: tasks [last, nt)
        flow, mask = (x.clone() for x in eng.debug_state(nt - last))
        for i in range(nt):
            one = eng.forward(fr, f0[i:i + 1], f1[i:i + 1], ts[i:i + 1], scale_factor=sf)
            assert torch.equal(got[i], one[0]), f"task {i} (pair {f0[i]}->{f1[i]}, t={ts[i]:.3f}) differs"
        eng.forward(fr, f0[last:], f1[last:], ts[last:], scale_factor=sf)
        flow1, mask1 = eng.debug_state(nt - last)
        assert torch.equal(flow, flow1) and torch.equal(mask, mask1), "debug state is not the last pass's"
    finally:
        eng.close()


@pytest.mark.parametrize("operand", ["float16", "bfloat16"])
@pytest.mark.parametrize("arch", ["4.6", "4.7", "4.17", "4.26"])
def test_layer_plans_unchanged(pkg, arch, operand):
    from cfi_b200.engine import Rife46Engine
    with open(os.path.join(ROOT, "tests", "golden", "rife_layer_plans.json")) as fh:
        plans = json.load(fh)
    eng = Rife46Engine(O.synthetic_state_dict(17, arch=arch), 0, operand, arch=arch)
    try:
        for b, layers in enumerate(plans[arch][operand]):
            for l, row in enumerate(layers):
                p = eng.layer_plan(b, l)
                assert [int(p[k]) for k in plans["fields"]] == row, (arch, operand, b, l, p)
    finally:
        eng.close()
