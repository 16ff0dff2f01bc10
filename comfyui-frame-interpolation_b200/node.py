"""ComfyUI node surface of the H100 path: a drop-in for the reference's `RIFE VFI` node.

Mirrors vfi_models/rife/__init__.py:34-239 (class attributes, kwargs, task order, skip / multiplier-list
semantics, output assembly, dtype round trip) and vfi_utils.py:49-81, :391-407 (InterpolationStateList,
MakeInterpolationStateList, FloatToInt).  The per-batch hot loop (:185-222) is replaced by ONE call into
libvfi_b200.so per GPU; there is no PyTorch/CPU fallback.

Host memory.  `frames` is taken as it comes (a ComfyUI IMAGE is a pageable CPU tensor): the library stages it
through a small ring of pinned buffers (csrc/hoststage.h), nothing of the caller's is pinned or copied here.
The output is allocated page-locked through torch's caching host allocator - its block is reused by the next call
once the previous result has been dropped, so only the first call pays for the allocation - up to
VFI_PINNED_OUT_MAX_GB (default 8); larger results are ordinary pageable tensors that the library fills through its
pinned download ring.

Several GPUs in one process.  set_devices([0, 1, ...]) (or VFI_DEVICES="0,1,2,3" / "all") shards the (pair, timestep)
task list over the listed devices: one engine (vfi_ctx) and one host thread per device, each with a contiguous,
task-count-balanced slice and only its own frame range, every device writing its frames straight into their slots
of the shared output tensor - no gather (rife/__init__.py:185-222 is one loop on one device).
"""
import collections
import os
import pathlib
import threading
import typing

import torch

from .engine import Rife46Engine, host_copy_frames

MODEL_TYPE = "rife"
# The reference table (rife/__init__.py:10-20) has no 4.6 entry at this commit although IFNet supports it and
# GMFSS uses rife46.pth (SURVEY.md F3); this node adds it.  Built archs: 4.6, 4.7 (rife47/rife49, the reference's
# default), 4.17 and 4.26; arch 4.0 (sudo_rife4, with contextnet/unet) is not built and raises KeyError here.
CKPT_NAME_VER_DICT = {
    "rife46.pth": "4.6",
    "rife47.pth": "4.7",
    "rife49.pth": "4.7",
    "rife417.pth": "4.17",
    "rife426.pth": "4.26",
}
DTYPE_OPTIONS = ["float32", "float16", "bfloat16"]
DTYPE_MAP = {"float32": torch.float32, "float16": torch.float16, "bfloat16": torch.bfloat16}

# (ckpt_name, dtype, device) -> engine, most recently used last.  An engine owns a multi-GB device workspace, so the
# cache is bounded (VFI_MODEL_CACHE entries per device, default 2) and evicted engines are closed.
_model_cache: "collections.OrderedDict[typing.Tuple, Rife46Engine]" = collections.OrderedDict()
_devices: typing.Optional[typing.List[int]] = None


def set_devices(devices: typing.Optional[typing.Sequence[int]]):
    """GPUs the node shards a clip over (None: the current device only, like the reference)."""
    global _devices
    _devices = None if devices is None else list(dict.fromkeys(int(d) for d in devices))


def _device_list() -> typing.List[int]:
    if _devices is not None:
        return list(_devices)
    env = os.environ.get("VFI_DEVICES", "").strip()
    if env == "all":
        return list(range(torch.cuda.device_count()))
    if env:
        return list(dict.fromkeys(int(x) for x in env.split(",") if x.strip() != ""))  # (an engine serves one thread)
    return [torch.cuda.current_device()]


def _engine_for(ckpt_name, dtype, device, arch_ver, model_path) -> Rife46Engine:
    key = (ckpt_name, dtype, int(device))
    eng = _model_cache.get(key)
    if eng is None:
        sd = torch.load(model_path, map_location="cpu", weights_only=False)
        eng = Rife46Engine(sd, device=int(device), dtype=dtype, arch=arch_ver)
        _model_cache[key] = eng
        cap = max(1, int(os.environ.get("VFI_MODEL_CACHE", "2")))
        on_dev = [k for k in _model_cache if k[2] == int(device)]
        for k in on_dev[:-cap]:
            _model_cache.pop(k).close()
    else:
        _model_cache.move_to_end(key)
    return eng


def clear_model_cache():
    while _model_cache:
        _model_cache.popitem()[1].close()


def _alloc_output(shape) -> torch.Tensor:
    nbytes = 4
    for d in shape:
        nbytes *= int(d)
    cap = float(os.environ.get("VFI_PINNED_OUT_MAX_GB", "8")) * (1 << 30)
    return torch.empty(shape, dtype=torch.float32, pin_memory=bool(torch.cuda.is_available() and nbytes <= cap))


class InterpolationStateList:
    """vfi_utils.py:49-57"""

    def __init__(self, frame_indices: typing.List[int], is_skip_list: bool):
        self.frame_indices = frame_indices
        self.is_skip_list = is_skip_list

    def is_frame_skipped(self, frame_index):
        is_frame_in_list = frame_index in self.frame_indices
        return self.is_skip_list and is_frame_in_list or not self.is_skip_list and not is_frame_in_list


class MakeInterpolationStateList:
    """vfi_utils.py:60-81"""

    @classmethod
    def INPUT_TYPES(s):
        return {
            "required": {
                "frame_indices": ("STRING", {"multiline": True, "default": "1,2,3"}),
                "is_skip_list": ("BOOLEAN", {"default": True},),
            },
        }

    RETURN_TYPES = ("INTERPOLATION_STATES",)
    FUNCTION = "create_options"
    CATEGORY = "ComfyUI-Frame-Interpolation/VFI"

    def create_options(self, frame_indices: str, is_skip_list: bool):
        frame_indices_list = [int(item) for item in frame_indices.split(',')]
        return (InterpolationStateList(frame_indices=frame_indices_list, is_skip_list=is_skip_list),)


class FloatToInt:
    """vfi_utils.py:391-407"""

    @classmethod
    def INPUT_TYPES(s):
        return {"required": {"float": ("FLOAT", {"default": 0, 'min': 0, 'step': 0.01})}}

    RETURN_TYPES = ("INT",)
    FUNCTION = "convert"
    CATEGORY = "ComfyUI-Frame-Interpolation"

    def convert(self, float):
        if hasattr(float, "__iter__"):
            return (list(map(int, float)),)
        return (int(float),)


def get_ckpt_container_path(model_type):
    root = os.environ.get("VFI_CKPT_DIR") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "ckpts")
    return os.path.abspath(os.path.join(root, model_type))


def load_file_from_github_release(model_type, ckpt_name):
    """Same role and name as vfi_utils.py:118-133, minus the download: the file must already be in
    <ckpts>/<model_type>/ (default ./ckpts, or $VFI_CKPT_DIR), exactly where the reference caches it."""
    path = os.path.join(get_ckpt_container_path(model_type), ckpt_name)
    if not os.path.exists(path):
        raise Exception(f"{ckpt_name} not found at {path}; copy the checkpoint there (this build never downloads)")
    return path


def build_tasks(n_pairs, multiplier, optional_interpolation_states):
    """Flat (pair_idx, timestep) list - rife/__init__.py:149-174."""
    if isinstance(multiplier, int):
        multipliers = [int(multiplier)] * n_pairs
    else:
        multipliers = list(map(int, multiplier))
        multipliers += [2] * (n_pairs - len(multipliers))
    tasks: typing.List[typing.Tuple[int, float]] = []
    for pair_idx in range(n_pairs):
        if optional_interpolation_states is not None and optional_interpolation_states.is_frame_skipped(pair_idx):
            continue
        m = multipliers[pair_idx]
        for step in range(1, m):
            tasks.append((pair_idx, step / m))
    return tasks, multipliers


class RIFE_VFI:
    @classmethod
    def INPUT_TYPES(s):
        return {
            "required": {
                "ckpt_name": (sorted(list(CKPT_NAME_VER_DICT.keys())), {"default": "rife49.pth"}),
                "frames": ("IMAGE",),
                "clear_cache_after_n_frames": ("INT", {"default": 10, "min": 1, "max": 1000}),
                "multiplier": ("INT", {"default": 2, "min": 1}),
                "fast_mode": ("BOOLEAN", {"default": True}),
                "ensemble": ("BOOLEAN", {"default": True}),
                "scale_factor": ([0.25, 0.5, 1.0, 2.0, 4.0], {"default": 1.0}),
                "dtype": (DTYPE_OPTIONS, {"default": "float32"}),
                "torch_compile": ("BOOLEAN", {"default": False}),
                "batch_size": ("INT", {"default": 1, "min": 1, "max": 64}),
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
        clear_cache_after_n_frames: int = 10,
        multiplier: typing.SupportsInt = 2,
        fast_mode: bool = False,
        ensemble: bool = False,
        scale_factor: float = 1.0,
        dtype: str = "float32",
        torch_compile: bool = False,
        batch_size: int = 1,
        optional_interpolation_states: InterpolationStateList = None,
        **kwargs
    ):
        """Same contract as the reference: frames [N,H,W,C] float32 in [0,1] -> ([(N-1)*m+1, H, W, 3] float32 CPU,).

        Accepted for API compatibility, without effect on results: clear_cache_after_n_frames (the workspace is
        pre-allocated, nothing to clear), fast_mode / ensemble (they never reach the 4.6 maths in the reference
        either - positional mis-wiring, SURVEY.md F7), torch_compile, batch_size (internal passes are sized by
        the engine).  all five scale_factor values work for every checkpoint.  dtype selects the tensor-core operand type: float32/float16 -> fp16 operands with fp32
        accumulation (same 10-bit mantissa as the TF32 convs the reference's float32 mode runs on a GPU),
        bfloat16 -> bf16 operands; flow, mask, warps and blending are fp32 in every mode.
        """
        arch_ver = CKPT_NAME_VER_DICT[ckpt_name]
        model_path = load_file_from_github_release(MODEL_TYPE, ckpt_name)
        torch_dtype = DTYPE_MAP[dtype]
        devices = _device_list()
        engines = [_engine_for(ckpt_name, dtype, d, arch_ver, model_path) for d in devices]

        assert len(frames) >= 2, f"RIFE needs at least 2 frames, only found {frames.shape[0]}"
        frames = frames.detach()
        # borrowed, never mutated; a CPU float32 contiguous IMAGE (the normal case) is used in place, pageable or not
        src = frames.to("cpu", torch.float32).contiguous()
        n, h, w, _ = src.shape
        n_pairs = n - 1
        tasks, _ = build_tasks(n_pairs, multiplier, optional_interpolation_states)

        # output order: each original frame followed by its interpolated frames - rife/__init__.py:225-231
        per_pair = [0] * n_pairs
        for p, _t in tasks:
            per_pair[p] += 1
        first_slot, slot = [], 0
        for p in range(n_pairs):
            first_slot.append(slot)
            slot += 1 + per_pair[p]
        total = slot + 1
        out = _alloc_output((total, h, w, 3))
        seen = [0] * n_pairs
        f0, f1, ts, slots = [], [], [], []
        for p, t in tasks:
            seen[p] += 1
            f0.append(p); f1.append(p + 1); ts.append(t); slots.append(first_slot[p] + seen[p])

        # one contiguous, task-count-balanced slice per device (skip lists / multiplier lists stay balanced); a device
        # uploads only the frames its slice touches and downloads straight into the slots of the shared output
        from .shard import shard_tasks
        jobs = [[e, lo, hi, None] for e, (lo, hi) in zip(engines, shard_tasks(len(tasks), len(engines))) if hi > lo]
        # pass-through frames (rife/__init__.py:227-231): every source frame also appears unchanged in the output.  The
        # library's copy threads put frame i into its slot while staging it for upload (one host copy for both); each
        # frame belongs to the first device whose frame range holds it, frames no device touches to the first device.
        orig_slots = first_slot + [total - 1]
        fast_pt = torch_dtype == torch.float32 and len(jobs) > 0
        if fast_pt:
            owner = [-1] * n
            for j, (_e, lo, hi, _) in enumerate(jobs):
                for f in range(min(f0[lo:hi]), max(f1[lo:hi]) + 1):
                    if owner[f] < 0:
                        owner[f] = j
            for j, job in enumerate(jobs):
                job[3] = [orig_slots[f] if owner[f] == j else -1 for f in range(n)]
        err: typing.List[BaseException] = []

        def run(engine, lo, hi, fslots):
            try:
                fr = (min(f0[lo:hi]), max(f1[lo:hi]) + 1)
                engine.interpolate_host(src, f0[lo:hi], f1[lo:hi], ts[lo:hi], out, out_slots=slots[lo:hi], frame_range=fr,
                                        scale_factor=float(scale_factor), frame_slots=fslots)
            except BaseException as e:  # surfaced on the caller's thread below
                err.append(e)

        threads = [threading.Thread(target=run, args=tuple(j)) for j in jobs]
        for th in threads:
            th.start()
        if fast_pt:
            rest = [orig_slots[f] if owner[f] < 0 else -1 for f in range(n)]  # frames of skipped pairs, never uploaded
            if any(v >= 0 for v in rest):
                host_copy_frames(src, rest, out)
        elif torch_dtype == torch.float32:
            host_copy_frames(src, orig_slots, out)
        else:  # the reference round-trips every frame through `dtype` (:227,:230,:238)
            out.index_copy_(0, torch.tensor(orig_slots, dtype=torch.long), src[..., :3].to(torch_dtype).to(torch.float32))
        for th in threads:
            th.join()
        if err:
            raise err[0]
        if torch_dtype != torch.float32 and slots:
            mid = torch.tensor(slots, dtype=torch.long)
            out.index_copy_(0, mid, out.index_select(0, mid).to(torch_dtype).to(torch.float32))
        return (out,)
