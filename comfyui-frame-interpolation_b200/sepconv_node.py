"""ComfyUI node surface of the H100 Sepconv path: a drop-in for the reference's `Sepconv VFI` node
(vfi_models/sepconv/__init__.py:13-57): same attributes and kwargs; the model call inside
`generic_frame_loop(..., use_timestep=False)` is `SepconvEngine.middle_frame` (libvfi_b200.so), no fallback."""
import typing

import torch

from .engine import SepconvEngine
from .frame_loop import generic_frame_loop
from .node import InterpolationStateList, load_file_from_github_release

MODEL_TYPE = "sepconv"
CKPT_NAMES = ["sepconv.pth"]
_model_cache: typing.Dict[str, SepconvEngine] = {}


def _load_engine(ckpt_name: str) -> SepconvEngine:
    if ckpt_name not in _model_cache:
        model_path = load_file_from_github_release(MODEL_TYPE, ckpt_name)
        sd = torch.load(model_path, map_location="cpu", weights_only=False)   # sepconv/__init__.py:44
        _model_cache[ckpt_name] = SepconvEngine(sd, device=torch.cuda.current_device(), dtype="float32")
    return _model_cache[ckpt_name]


PAIRS_PER_CALL = 2


def _vfi_x2_pipelined(engine: SepconvEngine, frames: torch.Tensor, states) -> torch.Tensor:
    """multiplier 2 (one middle frame per kept pair): the result of `generic_frame_loop(..., 2, ..., use_timestep=False)`
    (vfi_utils.py:260-337: every frame, followed by model(frame_i, frame_i+1) unless pair i is skipped; the last frame
    appended) without its per-pair synchronous `.to(device)` / `.cpu()` round trips: the frames stay in ComfyUI's NHWC
    layout (the engine reads it directly), source frames go up through two pinned staging buffers on a copy stream, middle
    frames come down on a third stream straight into their slots of the page-locked output while the next pairs compute."""
    from .node import _alloc_output
    dev = torch.device("cuda", engine.device)
    src = frames.detach()[..., :3].to("cpu", torch.float32).contiguous()
    n, h, w, _ = src.shape
    kept = [i for i in range(n - 1) if not (states is not None and states.is_frame_skipped(i))]
    kept_set = set(kept)
    first_slot, slot = [], 0
    for i in range(n - 1):
        first_slot.append(slot)
        slot += 2 if i in kept_set else 1
    total = slot + 1
    out = _alloc_output((total, h, w, 3))
    s_up, s_dn = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
    s_cp = torch.cuda.current_stream(dev)
    chunks = [kept[c:c + PAIRS_PER_CALL] for c in range(0, len(kept), PAIRS_PER_CALL)]
    stage = [torch.empty((2 * PAIRS_PER_CALL, h, w, 3), dtype=torch.float32).pin_memory() for _ in range(2)]
    dev_in = [torch.empty((2 * PAIRS_PER_CALL, h, w, 3), dtype=torch.float32, device=dev) for _ in range(2)]
    dev_out = [torch.empty((PAIRS_PER_CALL, h, w, 3), dtype=torch.float32, device=dev) for _ in range(2)]
    up_done = [torch.cuda.Event() for _ in range(2)]
    comp_done = [torch.cuda.Event() for _ in range(2)]
    dn_done = [torch.cuda.Event() for _ in range(2)]

    def upload(ci):
        b = ci & 1
        if ci >= 2:
            up_done[b].synchronize()       # the pinned buffer's previous copy has been read
        for j, i in enumerate(chunks[ci]):  # frames i and i + 1 of every pair of the chunk (host copy into pinned memory)
            stage[b][2 * j].copy_(src[i])
            stage[b][2 * j + 1].copy_(src[i + 1])
        with torch.cuda.stream(s_up):
            if ci >= 2:
                s_up.wait_event(comp_done[b])   # the device buffer's previous reader
            dev_in[b][: 2 * len(chunks[ci])].copy_(stage[b][: 2 * len(chunks[ci])], non_blocking=True)
            up_done[b].record(s_up)

    if chunks:
        upload(0)
    for ci, chunk in enumerate(chunks):
        b = ci & 1
        if ci + 1 < len(chunks):
            upload(ci + 1)                       # next chunk's host copy + H2D while this one computes
        s_cp.wait_event(up_done[b])
        if ci >= 2:
            s_cp.wait_event(dn_done[b])          # dev_out[b] has been downloaded
        k = len(chunk)
        engine.forward(dev_in[b], [2 * j for j in range(k)], [2 * j + 1 for j in range(k)], out=dev_out[b][:k])
        comp_done[b].record(s_cp)
        with torch.cuda.stream(s_dn):
            s_dn.wait_event(comp_done[b])
            for j, i in enumerate(chunk):
                out[first_slot[i] + 1].copy_(dev_out[b][j], non_blocking=True)
            dn_done[b].record(s_dn)
    # pass-through frames on the host while the GPU works
    from .engine import host_copy_frames
    host_copy_frames(src, first_slot + [total - 1], out)
    s_dn.synchronize()
    s_cp.synchronize()
    return out


class SepconvVFI:
    @classmethod
    def INPUT_TYPES(s):
        return {
            "required": {
                "ckpt_name": (CKPT_NAMES,),
                "frames": ("IMAGE",),
                "clear_cache_after_n_frames": ("INT", {"default": 10, "min": 1, "max": 1000}),
                "multiplier": ("INT", {"default": 2, "min": 2, "max": 1000})
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
        engine = kwargs.pop("_engine", None) or _load_engine(ckpt_name)
        # the pipelined path drives the library engine's device buffers; any other middle-frame model (a caller-supplied
        # engine) goes through the generic loop, whether or not a GPU is present
        if type(multiplier) == int and multiplier == 2 and frames.shape[0] >= 2 and isinstance(engine, SepconvEngine):
            return (_vfi_x2_pipelined(engine, frames, optional_interpolation_states),)
        x = frames[..., :3].permute(0, 3, 1, 2)   # preprocess_frames, vfi_utils.py:139-140

        def return_middle_frame(frame_0, frame_1, timestep, model):
            return model.middle_frame(frame_0, frame_1)

        out = generic_frame_loop(type(self).__name__, x, clear_cache_after_n_frames, multiplier, return_middle_frame, engine,
                                 interpolation_states=optional_interpolation_states, use_timestep=False,
                                 dtype=torch.float32)
        return (out.permute(0, 2, 3, 1),)   # postprocess_frames, vfi_utils.py:142-143
