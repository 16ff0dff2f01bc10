"""ComfyUI node surface of the H100 IFUnet path: a drop-in for the reference's `IFUnet VFI` node
(vfi_models/ifunet/__init__.py): the same class attributes, kwargs and defaults, the one checkpoint, and the pairs driven
through `generic_frame_loop` (use_timestep=True, dtype float32) with the model called by keyword, as the reference
does: ``model(frame_0, frame_1, timestep=timestep, scale=scale_factor, ensemble=ensemble)``.  The model call is
``IfunetEngine.forward`` (libvfi_b200.so kernels), one pair per call; there is no PyTorch / CPU fallback.

The checkpoint is read from <ckpts>/ifunet/ as the reference stores it: a raw ``IFUNetModel`` state dict, loaded
strictly.  A ``scale_factor`` at which the reference raises (most values other than 0.5, 1.0, 1.5, 2.0 .. 4.0; see
DESIGN.md section 12) raises a RuntimeError here too, before any kernel runs.
"""
import typing

import torch

from .engine import IfunetEngine
from .frame_loop import generic_frame_loop
from .node import InterpolationStateList, load_file_from_github_release

MODEL_TYPE = "ifunet"
CKPT_NAMES = ["IFUNet.pth"]

_model_cache: typing.Dict[str, IfunetEngine] = {}


def _load_engine(ckpt_name: str) -> IfunetEngine:
    if ckpt_name not in _model_cache:
        sd = torch.load(load_file_from_github_release(MODEL_TYPE, ckpt_name), map_location="cpu")
        _model_cache[ckpt_name] = IfunetEngine(sd, device=torch.cuda.current_device(), dtype="float32")
    return _model_cache[ckpt_name]


class IFUnet_VFI:
    @classmethod
    def INPUT_TYPES(s):
        return {
            "required": {
                "ckpt_name": (CKPT_NAMES, ),
                "frames": ("IMAGE", ),
                "clear_cache_after_n_frames": ("INT", {"default": 10, "min": 1, "max": 1000}),
                "multiplier": ("INT", {"default": 2, "min": 2, "max": 1000}),
                "scale_factor": ("FLOAT", {"default": 1.0, "min": 0.1, "max": 100, "step": 0.1}),
                "ensemble": ("BOOLEAN", {"default": True})
            },
            "optional": {
                "optional_interpolation_states": ("INTERPOLATION_STATES", )
            }
        }

    RETURN_TYPES = ("IMAGE", )
    FUNCTION = "vfi"
    CATEGORY = "ComfyUI-Frame-Interpolation/VFI"

    def vfi(
        self,
        ckpt_name: typing.AnyStr,
        frames: torch.Tensor,
        clear_cache_after_n_frames: typing.SupportsInt = 1,
        multiplier: typing.SupportsInt = 2,
        scale_factor: typing.SupportsFloat = 1.0,
        ensemble: bool = True,
        optional_interpolation_states: InterpolationStateList = None,
        **kwargs
    ):
        engine = kwargs.pop("_engine", None) or _load_engine(ckpt_name)
        dev = getattr(engine, "torch_device", None) or torch.device("cuda", engine.device)
        x = frames[..., :3].permute(0, 3, 1, 2)   # preprocess_frames, vfi_utils.py:139-140

        def return_middle_frame(frame_0, frame_1, timestep, model, scale_factor, ensemble):
            f0 = frame_0.to(dev, torch.float32).contiguous()
            f1 = frame_1.to(dev, torch.float32).contiguous()
            return model.forward(f0, f1, timestep=float(timestep), scale=float(scale_factor), ensemble=bool(ensemble))

        out = generic_frame_loop(type(self).__name__, x, clear_cache_after_n_frames, multiplier, return_middle_frame,
                                 engine, scale_factor, ensemble, interpolation_states=optional_interpolation_states,
                                 dtype=torch.float32)
        return (out.permute(0, 2, 3, 1)[..., :3].cpu(),)   # postprocess_frames, vfi_utils.py:142-143
