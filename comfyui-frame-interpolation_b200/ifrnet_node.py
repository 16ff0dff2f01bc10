"""ComfyUI node surface of the H100 IFRNet path: a drop-in for the reference's `IFRNet VFI` node
(vfi_models/ifrnet/__init__.py): the same class attributes, kwargs and defaults, the four checkpoints, IFRNet-S or
IFRNet-L by ``'S' in ckpt_name``, and the pairs driven through `generic_frame_loop` (use_timestep=True) as the GMFSS node
does.  The model call is ``IfrnetEngine.forward`` (libvfi_b200.so kernels); there is no PyTorch / CPU fallback.

The reference swaps two arguments, and this node keeps the swap: ``return_middle_frame(f0, f1, timestep, model,
scale_factor)`` calls ``model(f0, f1, timestep, scale_factor)`` against ``forward(img0, img1, scale_factor=1.0,
timestep=0.5)``.  So the loop's timestep k / m is the factor the frames are resized by before the encoder, and the
node's ``scale_factor`` (0.25 .. 4.0) is the value of decoder 4's time plane ``embt``.  At the default multiplier 2 the
model runs on half-resolution inputs with embt = 1.0; at multiplier 3 the two middles run at 1/3 and 2/3 of the padded
resolution.  The reference's output sizes at such factors are reproduced, not corrected (DESIGN.md section 10).
"""
import typing

import torch

from .engine import IfrnetEngine
from .frame_loop import generic_frame_loop
from .node import InterpolationStateList, load_file_from_github_release

MODEL_TYPE = "ifrnet"
CKPT_NAMES = ["IFRNet_S_Vimeo90K.pth", "IFRNet_L_Vimeo90K.pth", "IFRNet_S_GoPro.pth", "IFRNet_L_GoPro.pth"]

_model_cache: typing.Dict[str, IfrnetEngine] = {}


def _load_engine(ckpt_name: str) -> IfrnetEngine:
    if ckpt_name not in _model_cache:
        sd = torch.load(load_file_from_github_release(MODEL_TYPE, ckpt_name), map_location="cpu")
        eng = IfrnetEngine(sd, device=torch.cuda.current_device(), dtype="float32")
        want = "S" if "S" in ckpt_name else "L"
        if eng.variant != want:
            raise ValueError(f"{ckpt_name} holds IFRNet-{eng.variant} weights; the node builds IFRNet-{want} for this name")
        _model_cache[ckpt_name] = eng
    return _model_cache[ckpt_name]


class IFRNet_VFI:
    @classmethod
    def INPUT_TYPES(s):
        return {
            "required": {
                "ckpt_name": (CKPT_NAMES, ),
                "frames": ("IMAGE", ),
                "clear_cache_after_n_frames": ("INT", {"default": 10, "min": 1, "max": 1000}),
                "multiplier": ("INT", {"default": 2, "min": 2, "max": 1000}),
                "scale_factor": ([0.25, 0.5, 1.0, 2.0, 4.0], {"default": 1.0}),
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
        optional_interpolation_states: InterpolationStateList = None,
        **kwargs
    ):
        engine = kwargs.pop("_engine", None) or _load_engine(ckpt_name)
        dev = getattr(engine, "torch_device", None) or torch.device("cuda", engine.device)
        x = frames[..., :3].permute(0, 3, 1, 2)   # preprocess_frames, vfi_utils.py:139-140

        def return_middle_frame(frame_0, frame_1, timestep, model, scale_factor):
            f0 = frame_0.to(dev, torch.float32).contiguous()
            f1 = frame_1.to(dev, torch.float32).contiguous()
            # the reference's positional call: the timestep lands on the resize factor, scale_factor on embt
            return model.forward(f0, f1, float(timestep), float(scale_factor))

        out = generic_frame_loop(type(self).__name__, x, clear_cache_after_n_frames, multiplier, return_middle_frame,
                                 engine, scale_factor, interpolation_states=optional_interpolation_states,
                                 dtype=torch.float32)
        return (out.permute(0, 2, 3, 1)[..., :3].cpu(),)   # postprocess_frames, vfi_utils.py:142-143
