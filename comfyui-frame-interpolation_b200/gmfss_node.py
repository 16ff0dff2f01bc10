"""ComfyUI node surface of the H100 GMFSS Fortuna path: a drop-in for the reference's `GMFSS Fortuna VFI` node
(vfi_models/gmfss_fortuna/__init__.py:79-143): same attributes and kwargs; the model call inside
`generic_frame_loop(..., use_timestep=True)` is `gmfss.GMFSS.interpolate` (libvfi_b200.so kernels), no fallback.
Both checkpoints of the reference's dropdown are served: `GMFSS_fortuna_union` (five files, with the RIFE 4.6 sub-model; the
configuration SURVEY.md section 8 / BASELINE.json configs[3] name) and `GMFSS_fortuna` (four files, the base model without
it); `gmfss.build_gpu_model` tells them apart by the presence of `ifnet`."""
import typing

import torch

from .frame_loop import generic_frame_loop
from .node import InterpolationStateList, load_file_from_github_release

GLOBAL_MODEL_TYPE = "gmfss_fortuna"
# gmfss_fortuna/__init__.py:11-25
CKPTS_PATH_CONFIG = {
    "GMFSS_fortuna_union": {
        "ifnet": ("rife", "rife46.pth"),
        "flownet": (GLOBAL_MODEL_TYPE, "GMFSS_fortuna_flownet.pkl"),
        "metricnet": (GLOBAL_MODEL_TYPE, "GMFSS_fortuna_union_metric.pkl"),
        "feat_ext": (GLOBAL_MODEL_TYPE, "GMFSS_fortuna_union_feat.pkl"),
        "fusionnet": (GLOBAL_MODEL_TYPE, "GMFSS_fortuna_union_fusionnet.pkl"),
    },
    "GMFSS_fortuna": {
        "flownet": (GLOBAL_MODEL_TYPE, "GMFSS_fortuna_flownet.pkl"),
        "metricnet": (GLOBAL_MODEL_TYPE, "GMFSS_fortuna_metric.pkl"),
        "feat_ext": (GLOBAL_MODEL_TYPE, "GMFSS_fortuna_feat.pkl"),
        "fusionnet": (GLOBAL_MODEL_TYPE, "GMFSS_fortuna_fusionnet.pkl"),
    },
}
_model_cache: typing.Dict[str, typing.Any] = {}


def _strip(sd):
    """the reference's convert() (GMFSS_Fortuna_union_arch.py:1701-1706): checkpoints saved from DataParallel carry 'module.'"""
    return {k.replace("module.", ""): v for k, v in sd.items()}


def _load_model(ckpt_name: str):
    if ckpt_name not in _model_cache:
        from .gmfss import build_gpu_model
        cfg = CKPTS_PATH_CONFIG[ckpt_name]
        sds = {key: _strip(torch.load(load_file_from_github_release(*cfg[key]), map_location="cpu", weights_only=False)) for key in cfg}
        _model_cache[ckpt_name] = build_gpu_model(sds, torch.cuda.current_device())
    return _model_cache[ckpt_name]


class GMFSS_Fortuna_VFI:
    @classmethod
    def INPUT_TYPES(s):
        return {
            "required": {
                "ckpt_name": (list(CKPTS_PATH_CONFIG.keys()),),
                "frames": ("IMAGE",),
                "clear_cache_after_n_frames": ("INT", {"default": 10, "min": 1, "max": 1000}),
                "multiplier": ("INT", {"default": 2, "min": 2, "max": 1000}),
            },
            "optional": {
                "optional_interpolation_states": ("INTERPOLATION_STATES",)
            }
        }

    RETURN_TYPES = ("IMAGE",)
    FUNCTION = "vfi"
    CATEGORY = "ComfyUI-Frame-Interpolation/VFI"

    def vfi(
        self,
        ckpt_name: typing.AnyStr,
        frames: torch.Tensor,
        clear_cache_after_n_frames=10,
        multiplier: typing.SupportsInt = 2,
        optional_interpolation_states: InterpolationStateList = None,
        **kwargs
    ):
        model = kwargs.pop("_model", None) or _load_model(ckpt_name)
        dev = model.o.dev
        x = frames[..., :3].permute(0, 3, 1, 2)   # preprocess_frames, vfi_utils.py:139-140

        def return_middle_frame(frame_0, frame_1, timestep, model):
            f0 = frame_0.to(dev, torch.float32).contiguous()
            f1 = frame_1.to(dev, torch.float32).contiguous()
            return model.interpolate(f0, f1, float(timestep))

        out = generic_frame_loop(type(self).__name__, x, clear_cache_after_n_frames, multiplier, return_middle_frame, model,
                                 interpolation_states=optional_interpolation_states, use_timestep=True, dtype=torch.float32)
        return (out.permute(0, 2, 3, 1),)   # postprocess_frames, vfi_utils.py:142-143
