"""ComfyUI node surface of the H100 CAIN path: a drop-in for the reference's `CAIN VFI` node
(vfi_models/cain/__init__.py): the same class attributes, kwargs and defaults, the one checkpoint, and the pairs driven
through `generic_frame_loop` with use_timestep=False, so multipliers above 2 bisect recursively at midpoints.  The model
call is ``CainEngine.forward`` (libvfi_b200.so kernels), one pair per call; there is no PyTorch / CPU fallback.

The checkpoint is read from <ckpts>/cain/ as the reference stores it: ``torch.load(path)["state_dict"]`` with the
``module.`` prefix of its keys stripped.  The middle frame is not clamped, as in the reference.
"""
import typing

import torch

from .engine import CainEngine
from .frame_loop import generic_frame_loop
from .node import InterpolationStateList, load_file_from_github_release

MODEL_TYPE = "cain"
CKPT_NAMES = ["pretrained_cain.pth"]

_model_cache: typing.Dict[str, CainEngine] = {}


def _load_engine(ckpt_name: str) -> CainEngine:
    if ckpt_name not in _model_cache:
        sd = torch.load(load_file_from_github_release(MODEL_TYPE, ckpt_name), map_location="cpu")["state_dict"]
        sd = {key.replace("module.", ""): value for key, value in sd.items()}
        _model_cache[ckpt_name] = CainEngine(sd, device=torch.cuda.current_device(), dtype="float32")
    return _model_cache[ckpt_name]


class CAIN_VFI:
    @classmethod
    def INPUT_TYPES(s):
        return {
            "required": {
                "ckpt_name": (CKPT_NAMES, ),
                "frames": ("IMAGE", ),
                "clear_cache_after_n_frames": ("INT", {"default": 10, "min": 1, "max": 1000}),
                "multiplier": ("INT", {"default": 2, "min": 2, "max": 1000})
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
        optional_interpolation_states: InterpolationStateList = None,
        **kwargs
    ):
        engine = kwargs.pop("_engine", None) or _load_engine(ckpt_name)
        dev = getattr(engine, "torch_device", None) or torch.device("cuda", engine.device)
        x = frames[..., :3].permute(0, 3, 1, 2)   # preprocess_frames, vfi_utils.py:139-140

        def return_middle_frame(frame_0, frame_1, timestep, model):
            f0 = frame_0.to(dev, torch.float32).contiguous()
            f1 = frame_1.to(dev, torch.float32).contiguous()
            return model.forward(f0, f1)

        out = generic_frame_loop(type(self).__name__, x, clear_cache_after_n_frames, multiplier, return_middle_frame,
                                 engine, interpolation_states=optional_interpolation_states, use_timestep=False,
                                 dtype=torch.float32)
        return (out.permute(0, 2, 3, 1)[..., :3].cpu(),)   # postprocess_frames, vfi_utils.py:142-143
