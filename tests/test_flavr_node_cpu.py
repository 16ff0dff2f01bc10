"""The FLAVR node's surface, window schedule and output assembly on the CPU: FLAVR_VFI.vfi with a fake engine that runs
the CPU oracle (oracle/flavr.py) against the unmodified reference node's outputs (tests/golden/flavr_node_*.npz), the
checkpoint table, the loader's `module.` prefix handling, and the four-frame minimum."""
import math
import os
import sys
import warnings

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden_flavr import flavr_cases, flavr_inputs  # noqa: E402
from oracle import flavr as OV  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


class OracleEngine:
    """FlavrEngine.forward on the CPU: window k -> oracle output 0 of frames first[k] .. first[k] + 3."""
    torch_device = torch.device("cpu")

    def __init__(self, sd):
        self.sd = sd
        self.calls = []

    def forward(self, frames, first):
        self.calls.append(list(first))
        return torch.stack([OV.interpolate(self.sd, frames[f:f + 4, ..., :3]) for f in first])


def psnr(a, b):
    mse = float(((a.double() - b.double()) ** 2).mean())
    return 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)


@pytest.mark.parametrize("name", [k for k, v in flavr_cases().items() if v["kind"] == "node"])
def test_node_matches_reference_node(pkg, name):
    import cfi_b200.flavr_node as FN
    cfg = flavr_cases()[name]
    ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
    eng = OracleEngine(OV.synthetic_state_dict(cfg["seed"], cfg["variant"]))
    st = None if cfg["states"] is None else FN.InterpolationStateList(list(cfg["states"][0]), cfg["states"][1])
    fr = flavr_inputs(cfg)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        (out,) = FN.FLAVR_VFI().vfi(cfg["ckpt"], fr, multiplier=cfg["multiplier"],
                                    duplicate_first_last_frames=cfg["dup"], optional_interpolation_states=st, _engine=eng)
    warned = any("FLAVR only supports 2x" in str(w.message) for w in caught)
    assert warned == (cfg["multiplier"] != 2)
    assert out.shape == ref.shape
    assert psnr(out, ref) >= 50.0
    # pass-through frames are the source frames bit for bit; only the new frames come from the model
    _, entries = FN.output_schedule(cfg["n"], cfg["dup"], st)
    for j, (kind, i) in enumerate(entries):
        if kind == "frame":
            assert torch.equal(out[j], ref[j]) and torch.equal(out[j], fr[i, ..., :3])
    # windows run in passes of at most WINDOWS_PER_PASS, each window once, in order
    assert all(len(c) <= FN.WINDOWS_PER_PASS for c in eng.calls)
    assert sum(eng.calls, []) == [i for i in range(cfg["n"] - 3)
                                   if not (st is not None and st.is_frame_skipped(i) and st.is_frame_skipped(i + 1))]


def test_schedule_drops_frames_of_skipped_first_and_last_window(pkg):
    import cfi_b200.flavr_node as FN
    st = FN.InterpolationStateList([0, 1, 3, 4], True)   # windows 0 and 3 of a 7-frame clip are skipped
    windows, entries = FN.output_schedule(7, True, st)
    assert windows == [1, 2]
    assert entries == [("new", 0), ("frame", 3), ("new", 1), ("frame", 4)]
    windows, entries = FN.output_schedule(4, True, None)
    assert entries == [("frame", 0), ("frame", 0), ("frame", 1), ("new", 0), ("frame", 2), ("frame", 3), ("frame", 3)]


def test_node_surface_and_registration(pkg):
    import cfi_b200 as P
    import cfi_b200.flavr_node as FN
    it = FN.FLAVR_VFI.INPUT_TYPES()
    assert it["required"]["ckpt_name"] == (["FLAVR_2x.pth", "FLAVR_4x.pth", "FLAVR_8x.pth"],)
    assert it["required"]["multiplier"] == ("INT", {"default": 2, "min": 2, "max": 2})
    assert it["required"]["duplicate_first_last_frames"] == ("BOOLEAN", {"default": False})
    assert it["required"]["clear_cache_after_n_frames"] == ("INT", {"default": 10, "min": 1, "max": 1000})
    assert it["optional"] == {"optional_interpolation_states": ("INTERPOLATION_STATES",)}
    assert FN.FLAVR_VFI.CATEGORY == "ComfyUI-Frame-Interpolation/VFI" and FN.FLAVR_VFI.FUNCTION == "vfi"
    assert FN.FLAVR_VFI.RETURN_TYPES == ("IMAGE",)
    assert P.NODE_CLASS_MAPPINGS["FLAVR VFI"] is FN.FLAVR_VFI
    assert P.NODE_DISPLAY_NAME_MAPPINGS["FLAVR VFI"] == "FLAVR VFI (H100 native)"


def test_fewer_than_four_frames_raise(pkg):
    import cfi_b200.flavr_node as FN
    eng = OracleEngine(OV.synthetic_state_dict(0, "2x"))
    with pytest.raises(AssertionError, match="at least 4 frames"):
        FN.FLAVR_VFI().vfi("FLAVR_2x.pth", torch.rand(3, 16, 16, 3), _engine=eng)
    assert eng.calls == []


@pytest.mark.parametrize("ckpt", ["FLAVR_2x.pth", "FLAVR_4x.pth", "FLAVR_8x.pth"])
def test_checkpoint_table_and_loader(pkg, monkeypatch, tmp_path, ckpt):
    """Each checkpoint loads from <ckpts>/flavr/ with the `module.` prefix stripped; its variant (outputs, encoder bias)
    is what the state dict says, and the names are the ones the engine passes to the library."""
    import cfi_b200.flavr_node as FN
    from cfi_b200.engine import flavr_state_dict_names
    variant = OV.CKPT_VARIANT[ckpt]
    n_out, bias = OV.VARIANTS[variant]
    sd = OV.synthetic_state_dict(7, variant)
    os.makedirs(tmp_path / "flavr")
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, tmp_path / "flavr" / ckpt)
    monkeypatch.setenv("VFI_CKPT_DIR", str(tmp_path))
    got = FN.load_state_dict(FN.load_file_from_github_release(FN.MODEL_TYPE, ckpt))
    assert list(got) == list(sd)
    assert got["outconv.1.weight"].shape[0] == 3 * n_out
    assert set(flavr_state_dict_names("encoder.stem.0.bias" in got)) == set(got)


def test_missing_checkpoint_is_an_error(pkg, monkeypatch, tmp_path):
    import cfi_b200.flavr_node as FN
    monkeypatch.setenv("VFI_CKPT_DIR", str(tmp_path))
    with pytest.raises(Exception, match="not found"):
        FN.load_file_from_github_release(FN.MODEL_TYPE, "FLAVR_2x.pth")
