"""ComfyUI node surface of the H100 FLAVR path: a drop-in for the reference's `FLAVR VFI` node.

Mirrors vfi_models/flavr/__init__.py:26-115: the class attributes and kwargs of ``FLAVR_VFI``, the warning for a
multiplier other than 2 (the node still interpolates 2x), the four-frame minimum, the sliding 4-frame window with its skip
rule (a window is skipped only when both of its first two frames are skipped, and a skipped first or last window also
drops the frames it would have appended) and the output order ``f0, [f0], f1`` / ``new, f2`` / ``f3, [f3]``.
``new`` is the model's first output, for the 4x / 8x checkpoints its t = 1/4 / 1/8 frame, not clamped.  The model call
is ``FlavrEngine.forward`` = one pass of libvfi_b200.so over up to ``WINDOWS_PER_PASS`` windows; there is no PyTorch /
CPU fallback.
"""
import typing
import warnings

import torch

from .engine import FlavrEngine
from .node import InterpolationStateList, _alloc_output, load_file_from_github_release

MODEL_TYPE = "flavr"
CKPT_NAMES = ["FLAVR_2x.pth", "FLAVR_4x.pth", "FLAVR_8x.pth"]
WINDOWS_PER_PASS = 4  # windows interpolated together (about 5 GB of workspace per 1080p window)
NBR_FRAME = 4

_model_cache: typing.Dict[str, FlavrEngine] = {}


def load_state_dict(path: str) -> typing.Dict[str, torch.Tensor]:
    """build_flavr (flavr/__init__.py:14-16): torch.load(path)['state_dict'] with the `module.` prefix stripped."""
    sd = torch.load(path, map_location="cpu")["state_dict"]
    return {k.partition("module.")[-1]: v for k, v in sd.items()}


def _load_engine(ckpt_name: str) -> FlavrEngine:
    if ckpt_name not in _model_cache:
        sd = load_state_dict(load_file_from_github_release(MODEL_TYPE, ckpt_name))
        _model_cache[ckpt_name] = FlavrEngine(sd, device=torch.cuda.current_device(), dtype="float32")
    return _model_cache[ckpt_name]


def output_schedule(n: int, duplicate_first_last_frames: bool,
                    states: typing.Optional[InterpolationStateList]) -> typing.Tuple[typing.List[int], list]:
    """(windows run, entries): entries list the output frames in order, ("frame", i) for source frame i and ("new", k)
    for the k-th window run (flavr/__init__.py:72-97)."""
    windows, entries = [], []
    for i in range(n - 3):
        if states is not None and states.is_frame_skipped(i) and states.is_frame_skipped(i + 1):
            continue
        k = len(windows)
        windows.append(i)
        if i == 0:
            entries.append(("frame", 0))
            if duplicate_first_last_frames:
                entries.append(("frame", 0))
            entries.append(("frame", 1))
        entries += [("new", k), ("frame", i + 2)]
        if i == n - 4:
            entries.append(("frame", i + 3))
            if duplicate_first_last_frames:
                entries.append(("frame", i + 3))
    return windows, entries


class FLAVR_VFI:
    @classmethod
    def INPUT_TYPES(s):
        return {
            "required": {
                "ckpt_name": (CKPT_NAMES,),
                "frames": ("IMAGE",),
                "clear_cache_after_n_frames": ("INT", {"default": 10, "min": 1, "max": 1000}),
                "multiplier": ("INT", {"default": 2, "min": 2, "max": 2}),
                "duplicate_first_last_frames": ("BOOLEAN", {"default": False}),
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
        duplicate_first_last_frames: bool = False,
        optional_interpolation_states: InterpolationStateList = None,
        **kwargs
    ):
        """frames [N,H,W,C>=3] float32 -> ([M,H,W,3] float32 CPU,) exactly as the reference assembles it.
        clear_cache_after_n_frames is accepted without effect (the workspace is owned by the engine)."""
        if multiplier != 2:
            warnings.warn("Currently, FLAVR only supports 2x interpolation. The process will continue but please set "
                          "multiplier=2 afterward")
        assert len(frames) >= NBR_FRAME, (
            f"VFI model ST-MFNet requires at least {NBR_FRAME} frames to work with, only found {frames.shape[0]}. "
            "Please check the frame input using PreviewImage.")  # assert_batch_size, vfi_utils.py:145-147
        engine = kwargs.pop("_engine", None) or _load_engine(ckpt_name)
        dev = getattr(engine, "torch_device", None) or torch.device("cuda", engine.device)
        src = frames.detach()[..., :3].to("cpu", torch.float32).contiguous()  # preprocess_frames vfi_utils.py:139-140
        n, h, w, _ = src.shape
        windows, entries = output_schedule(n, duplicate_first_last_frames, optional_interpolation_states)
        if not entries:
            raise RuntimeError("FLAVR VFI: every window is skipped, there is no frame to output")
        pin = dev.type == "cuda"
        out = _alloc_output((len(entries), h, w, 3)) if pin else torch.empty((len(entries), h, w, 3), dtype=torch.float32)
        new_slot = {}
        for j, (kind, i) in enumerate(entries):
            if kind == "frame":
                out[j].copy_(src[i])  # the padded frame, unpadded again (flavr/__init__.py:88-97, :110)
            else:
                new_slot[i] = j
        if windows:
            dframes = src.to(dev, non_blocking=pin)
            for c0 in range(0, len(windows), WINDOWS_PER_PASS):
                chunk = windows[c0:c0 + WINDOWS_PER_PASS]
                mids = engine.forward(dframes, chunk)
                for k in range(len(chunk)):
                    out[new_slot[c0 + k]].copy_(mids[k], non_blocking=pin)
            if pin:
                torch.cuda.current_stream(dev).synchronize()
        return (out,)
