"""FILM node host logic on CPU: schedule, skip / multiplier-list semantics and output assembly of
comfyui-frame-interpolation_b200/film_node.py against the outputs of the unmodified reference node
(tests/golden/film_node_*.npz).  The model call is a stand-in here (the CPU oracle behind the engine's
``forward`` signature) - the product engine needs an H100 and is covered by the GPU tests."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden_film import film_cases, film_inputs  # noqa: E402
from oracle import film as OF  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


class OracleEngine:
    """Stand-in with FilmEngine.forward's contract, computing on the CPU with the oracle (tests only)."""
    torch_device = torch.device("cpu")

    def __init__(self, sd):
        self.sd = sd
        self.calls = []

    def forward(self, frames, f0, f1, clamp=False, out=None):
        self.calls.append(len(f0))
        res = []
        for a, b in zip(f0, f1):
            x0 = frames[a:a + 1].permute(0, 3, 1, 2)
            x1 = frames[b:b + 1].permute(0, 3, 1, 2)
            y = OF.interpolator_forward(self.sd, x0, x1, torch.full((1, 1), 0.5))
            res.append((y.clamp(0, 1) if clamp else y).permute(0, 2, 3, 1))
        return torch.cat(res, 0)


@pytest.mark.parametrize("name", [n for n, c in sorted(film_cases().items()) if c["kind"] == "node"])
def test_film_node_matches_reference_node(pkg, name):
    import cfi_b200.film_node as FN
    cfg = film_cases()[name]
    ref = torch.from_numpy(np.load(os.path.join(GOLD, name + ".npz"))["out"])
    eng = OracleEngine(OF.synthetic_state_dict(cfg["seed"], cfg["flow_gain"]))
    st = None if cfg["states"] is None else FN.InterpolationStateList(list(cfg["states"][0]), cfg["states"][1])
    (out,) = FN.FILM_VFI().vfi("film_net_fp32.pt", film_inputs(cfg), multiplier=cfg["multiplier"],
                               optional_interpolation_states=st, _engine=eng)
    assert out.shape == ref.shape and out.dtype == torch.float32
    # the stand-in feeds NHWC-strided views to ATen (other conv kernels than for the reference's NCHW tensors) and the
    # recursion re-feeds its outputs: rounding-level differences only
    assert (out - ref).abs().max().item() <= 2e-5


def test_film_node_batches_pairs_with_equal_multipliers(pkg):
    import cfi_b200.film_node as FN
    eng = OracleEngine(OF.synthetic_state_dict(7))
    fr = OF.synthetic_clip(4, 64, 64, seed=3)
    (out,) = FN.FILM_VFI().vfi("film_net_fp32.pt", fr, multiplier=2, _engine=eng)
    assert eng.calls == [3]  # three pairs, one schedule step, one pass
    assert out.shape == (7, 64, 64, 3)
    for i in range(4):
        assert torch.equal(out[2 * i], fr[i])  # originals are passed through bit exact (film/__init__.py:96, :104)


def test_film_inference_order_matches_oracle(pkg):
    import cfi_b200.film_node as FN
    for k in (0, 1, 2, 3, 4, 5, 7, 9):
        assert FN.inference_order(k) == OF.inference_order(k)


def test_film_node_surface_matches_reference(pkg):
    """film/__init__.py:44-61 and root __init__.py:16, :34."""
    import cfi_b200 as P
    import cfi_b200.film_node as FN
    assert P.NODE_CLASS_MAPPINGS["FILM VFI"] is FN.FILM_VFI
    it = FN.FILM_VFI.INPUT_TYPES()
    assert list(it["required"].keys()) == ["ckpt_name", "frames", "clear_cache_after_n_frames", "multiplier"]
    assert it["required"]["ckpt_name"] == (["film_net_fp32.pt"],)
    assert it["required"]["multiplier"][1] == {"default": 2, "min": 2, "max": 1000}
    assert it["optional"] == {"optional_interpolation_states": ("INTERPOLATION_STATES",)}
    assert FN.FILM_VFI.RETURN_TYPES == ("IMAGE",) and FN.FILM_VFI.FUNCTION == "vfi"
    assert FN.FILM_VFI.CATEGORY == "ComfyUI-Frame-Interpolation/VFI"


def test_film_engine_names_match_oracle_spec(pkg):
    from cfi_b200.engine import film_state_dict_names
    assert film_state_dict_names() == [n for n, _ in OF.state_dict_spec()]


def test_film_no_gpu_is_a_loud_error(pkg):
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from cfi_b200._lib import VfiError
    from cfi_b200.engine import FilmEngine
    with pytest.raises(VfiError):
        FilmEngine(OF.synthetic_state_dict(0), 0)
