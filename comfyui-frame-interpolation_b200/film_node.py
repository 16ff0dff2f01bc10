"""ComfyUI node surface of the H100 FILM path: a drop-in for the reference's `FILM VFI` node.

Mirrors vfi_models/film/__init__.py:12-113: the class attributes and kwargs of ``FILM_VFI``, the bisection
schedule of ``inference`` (:12-42), the skip semantics (a skipped pair is dropped together with its first
frame, :85-86), the multiplier list padded with 2s (:81-83) and the output order (:96, :104-106).  The model
call (:35-38) is ``FilmEngine.forward`` = one pass of libvfi_b200.so over up to ``PAIRS_PER_PASS`` pairs that
are at the same step of their schedules; there is no PyTorch / CPU fallback.
"""
import bisect
import typing

import numpy as np
import torch

from .engine import FilmEngine
from .node import InterpolationStateList, _alloc_output, load_file_from_github_release

MODEL_TYPE = "film"
PAIRS_PER_PASS = 4  # pairs interpolated together (about 6 GB of workspace per 1080p pair)

_model_cache: typing.Dict[str, FilmEngine] = {}


def _load_engine(ckpt_name: str) -> FilmEngine:
    """film/__init__.py:73-77: the checkpoint is a TorchScript module; its state_dict carries the 82 tensors of
    film_arch.Interpolator."""
    if ckpt_name not in _model_cache:
        model_path = load_file_from_github_release(MODEL_TYPE, ckpt_name)
        sd = torch.jit.load(model_path, map_location="cpu").state_dict()
        _model_cache[ckpt_name] = FilmEngine(sd, device=torch.cuda.current_device(), dtype="float32")
    return _model_cache[ckpt_name]


def inference_order(inter_frames: int) -> typing.List[typing.Tuple[int, int, int]]:
    """The order in which film/__init__.py:12-42 creates the in-between frames, as (left, right, new) positions in
    the final sequence 0..inter_frames+1.  Same float32 arithmetic as the reference (torch.linspace / argmin), so
    ties between equally central candidates break the same way."""
    idxes = [0, inter_frames + 1]
    remains = list(range(1, inter_frames + 1))
    splits = torch.linspace(0, 1, inter_frames + 2)
    order = []
    for _ in range(len(remains)):
        starts = splits[idxes[:-1]]
        ends = splits[idxes[1:]]
        distances = ((splits[None, remains] - starts[:, None]) / (ends[:, None] - starts[:, None]) - .5).abs()
        matrix = torch.argmin(distances).item()
        start_i, step = np.unravel_index(matrix, distances.shape)
        end_i = start_i + 1
        order.append((idxes[start_i], idxes[end_i], remains[step]))
        idxes.insert(bisect.bisect_left(idxes, remains[step]), remains[step])
        del remains[step]
    return order


class FILM_VFI:
    @classmethod
    def INPUT_TYPES(s):
        return {
            "required": {
                "ckpt_name": (["film_net_fp32.pt"],),
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
        """frames [N,H,W,C>=3] float32 -> ([M,H,W,3] float32 CPU,) exactly as the reference assembles it.
        clear_cache_after_n_frames is accepted without effect (the workspace is owned by the engine)."""
        engine = kwargs.pop("_engine", None) or _load_engine(ckpt_name)
        dev = getattr(engine, "torch_device", None) or torch.device("cuda", engine.device)
        frames = frames.detach()
        src = frames[..., :3].to("cpu", torch.float32).contiguous()  # preprocess_frames vfi_utils.py:139-140
        n, h, w, _ = src.shape
        if type(multiplier) == int:
            multipliers = [multiplier] * n
        else:
            multipliers = list(map(int, multiplier))
            multipliers += [2] * (n - len(multipliers) - 1)
        pairs = [i for i in range(n - 1)
                 if not (optional_interpolation_states is not None and optional_interpolation_states.is_frame_skipped(i))]
        # output slots: every kept pair contributes its first frame + (multiplier - 1) new frames; the last frame closes
        # (a multiplier entry < 2 yields no new frame: `inference` returns the two inputs and [:-1] keeps the first)
        multipliers = [max(int(m), 1) for m in multipliers]
        first_slot, slot = {}, 0
        for i in pairs:
            first_slot[i] = slot
            slot += multipliers[i]
        total = slot + 1
        # page-locked through torch's caching host allocator up to VFI_PINNED_OUT_MAX_GB (node._alloc_output), pageable above
        pin = dev.type == "cuda"
        out = _alloc_output((total, h, w, 3)) if pin else torch.empty((total, h, w, 3), dtype=torch.float32)
        out[total - 1] = src[n - 1]
        # pairs with the same multiplier share a schedule and are interpolated PAIRS_PER_PASS at a time
        by_mult: typing.Dict[int, typing.List[int]] = {}
        for i in pairs:
            by_mult.setdefault(multipliers[i], []).append(i)
        for m, plist in by_mult.items():
            inter = m - 1
            order = inference_order(inter) if inter > 0 else []
            for c0 in range(0, len(plist), PAIRS_PER_PASS):
                chunk = plist[c0:c0 + PAIRS_PER_PASS]
                nc = len(chunk)
                # store[j, q]: frame at position q (0..inter+1) of the chunk's j-th pair
                store = torch.empty((nc, inter + 2, h, w, 3), dtype=torch.float32, device=dev)
                for j, i in enumerate(chunk):
                    store[j, 0].copy_(src[i], non_blocking=pin)
                    store[j, inter + 1].copy_(src[i + 1], non_blocking=pin)
                flat = store.view(nc * (inter + 2), h, w, 3)
                for lo, hi, new in order:
                    f0 = [j * (inter + 2) + lo for j in range(nc)]
                    f1 = [j * (inter + 2) + hi for j in range(nc)]
                    mid = engine.forward(flat, f0, f1, clamp=True)  # model(x0, x1, dt).clamp(0, 1), :35-38
                    store[:, new].copy_(mid)
                for j, i in enumerate(chunk):
                    out[first_slot[i]:first_slot[i] + m].copy_(store[j, :m], non_blocking=pin)  # relust[:-1], :96
                if pin:
                    torch.cuda.current_stream(dev).synchronize()
        return (out,)
