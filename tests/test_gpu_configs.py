"""-m gpu: parity AT THE CONFIGURATIONS THE NUMBERS ARE QUOTED ON (BASELINE.json configs[0] and configs[1]).

* config 1: the reference's demo pair (540 x 960) through the node mirror vs the unmodified reference node's output.
* config 2 geometry: 1080 x 1920 (padded 1088 x 1920), a pass of B = 8 pairs (the bench's internal batch: 132 persistent
  CTAs striding > 8 k tiles per layer) vs (a) the unmodified reference's crops / box-filtered frame and (b) the oracle's
  full frames computed on this box's CPU.
Tolerance (north_star): PSNR >= 50 dB on the interpolated frames; pass-through frames bit exact."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import rife46 as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden_configs import CFG1, CFG2, CROP, box8, crop_origins  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
QSTEP = 1.0 / 65535.0


@pytest.mark.parametrize("dtype", ["float32", "bfloat16"])
def test_config1_demo_pair_through_the_node(pkg, dtype, tmp_path, monkeypatch):
    import cfi_b200.node as N
    g = np.load(os.path.join(GOLD, "cfg1_anime_540p.npz"))
    fr = torch.from_numpy(g["frames_u8"]).float() / 255.0
    sd = O.synthetic_state_dict(CFG1["weight_seed"], CFG1["gain"], arch="4.6")
    path = tmp_path / "rife46.pth"
    torch.save(sd, path)
    monkeypatch.setattr(N, "load_file_from_github_release", lambda model_type, ckpt_name: str(path))
    N._model_cache.clear()
    (out,) = N.RIFE_VFI().vfi("rife46.pth", fr, multiplier=CFG1["multiplier"], dtype=dtype)
    N._model_cache.clear()
    assert out.shape == (3, 540, 960, 3) and out.dtype == torch.float32 and out.device.type == "cpu"
    if dtype == "float32":
        assert torch.equal(out[0], fr[0]) and torch.equal(out[2], fr[1])
    ref = torch.from_numpy(g["mid_q16"].astype(np.float32)) * QSTEP
    p = O.psnr(out[1], ref)
    print(f"config 1 (anime 540p, node, {dtype}): PSNR {p:.2f} dB")
    assert p >= 50.0


@pytest.mark.parametrize("arch", ["4.6", "4.7"])
def test_config2_geometry_1080p_batch8(pkg, arch):
    from cfi_b200.engine import Rife46Engine
    g = np.load(os.path.join(GOLD, "cfg2_1080p_arch" + arch.replace(".", "") + ".npz"))
    fr = O.synthetic_clip(2, CFG2["h"], CFG2["w"], seed=CFG2["clip_seed"])
    sd = O.synthetic_state_dict(CFG2["weight_seed"], CFG2["gain"], arch=arch)
    eng = Rife46Engine(sd, 0, "float32", batch=8)
    # one pass of 8 tasks over the same pair: the golden's two timesteps first, six more to fill the batch
    ts = list(CFG2["ts"]) + [0.125, 0.375, 0.625, 0.75, 0.875, 0.5]
    out = eng.forward(fr.cuda().contiguous(), [0] * 8, [1] * 8, ts).cpu()
    eng.close()
    assert out.shape == (8, CFG2["h"], CFG2["w"], 3)
    assert torch.equal(out[0], out[7]), "same task twice in one pass must give the same frame"
    o = out.numpy()
    crops = g["crops_q16"].astype(np.float32) * QSTEP
    mine = np.stack([o[:2, y:y + CROP, x0:x0 + CROP] for y, x0 in crop_origins(CFG2["h"], CFG2["w"])], 1)
    worst = min(O.psnr(torch.from_numpy(mine[:, i]), torch.from_numpy(crops[:, i])) for i in range(mine.shape[1]))
    p_crops = O.psnr(torch.from_numpy(mine), torch.from_numpy(crops))
    b8 = np.abs(box8(o[:2]) - g["box8_q16"].astype(np.float32) * QSTEP).max()
    # the oracle's full frames on this box's CPU (pinned to the reference at this size by tests/test_oracle_configs.py)
    x = fr.permute(0, 3, 1, 2)
    tt = torch.tensor(ts[2:4], dtype=torch.float32).view(-1, 1, 1, 1)
    ref = O.ifnet_forward(arch, sd, x[0:1].repeat(2, 1, 1, 1), x[1:2].repeat(2, 1, 1, 1), tt).clamp(0, 1).permute(0, 2, 3, 1)
    p_full = O.psnr(out[2:4], ref)
    print(f"config 2 geometry (1080p, B=8, arch {arch}): crops PSNR {p_crops:.2f} dB (worst crop {worst:.2f}), "
          f"8x8-box max abs {b8:.2e}, full frames vs oracle {p_full:.2f} dB")
    assert worst >= 50.0 and p_full >= 50.0 and b8 <= 2e-3


def test_node_shards_over_the_devices_of_this_process(pkg, tmp_path, monkeypatch):
    """set_devices: one engine + host thread per GPU, contiguous task slices, every device writing its own slots of the
    shared output (two GPUs when the box has them, else the same code path with one) == the single-device result."""
    import cfi_b200.node as N
    sd = O.synthetic_state_dict(3, 1.5, arch="4.6")
    path = tmp_path / "rife46.pth"
    torch.save(sd, path)
    monkeypatch.setattr(N, "load_file_from_github_release", lambda model_type, ckpt_name: str(path))
    fr = O.synthetic_clip(9, 72, 104, seed=31)
    st = N.InterpolationStateList([2], True)
    N._model_cache.clear()
    (one,) = N.RIFE_VFI().vfi("rife46.pth", fr, multiplier=[3, 2, 2, 4], optional_interpolation_states=st)
    devs = list(range(min(2, torch.cuda.device_count())))
    N.set_devices(devs)
    try:
        (two,) = N.RIFE_VFI().vfi("rife46.pth", fr, multiplier=[3, 2, 2, 4], optional_interpolation_states=st)
    finally:
        N.set_devices(None)
        N.clear_model_cache()
    assert torch.equal(one, two)
    ref = O.rife_vfi(sd, fr, multiplier=[3, 2, 2, 4], states=([2], True))
    assert one.shape == ref.shape and O.psnr(one, ref) >= 50.0
