"""The shared per-pair loop the reference's other nodes (GMFSS, Sepconv, M2M, IFRNet, ...) drive their models through:
`vfi_utils.generic_frame_loop` / `_generic_frame_loop` (vfi_utils.py:149-389), re-stated for this package so that a
H100 model function (frame0, frame1, timestep, *args) -> middle frame can be dropped behind any of those nodes.

Semantics kept (checked against the reference's own outputs, tests/golden/loop_*.npz):
  * int multiplier: every frame is emitted followed by its m-1 middles; a skipped pair keeps its first frame and
    emits no middles; the last frame is appended (vfi_utils.py:260-265, :329-337)
  * use_timestep=True : middle k uses timestep k/m (:203-211)
  * use_timestep=False: recursive midpoint bisection with n = m-1; even n drops the shared midpoint (:162-171)
  * list multiplier: padded with 2; each pair is looped on its own 2-frame clip, so the skip predicate sees pair
    index 0 for every pair (reference quirk, :364-388); multiplier 0 drops the pair including its first frame (:370)
  * outputs are CPU tensors of `dtype`, NCHW like the (pre-processed) input.
`batch_size` / `clear_cache_after_n_frames` are accepted and change nothing in the result (scheduling only).
"""
import typing

import torch


def _device():
    return torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")


def _bisect(fn, args, f0, f1, n):
    mid = fn(f0, f1, None, *args)
    if n == 1:
        return [mid]
    left = _bisect(fn, args, f0, mid, n // 2)
    right = _bisect(fn, args, mid, f1, n // 2)
    return left + ([mid] if n % 2 else []) + right


def _loop(frames, multiplier, fn, args, states, use_timestep, dtype):
    dev = _device()
    out = []
    for i in range(len(frames) - 1):
        f0, f1 = frames[i:i + 1], frames[i + 1:i + 2]
        out.append(f0.to(dtype=dtype))
        if states is not None and states.is_frame_skipped(i):
            continue
        a, b = f0.to(torch.float32).to(dev), f1.to(torch.float32).to(dev)
        if use_timestep:
            for k in range(1, multiplier):
                out.append(fn(a, b, k / multiplier, *args).detach().cpu().to(dtype=dtype))
        elif multiplier > 1:
            mids = _bisect(fn, args, a, b, multiplier - 1)
            out.extend(m.detach().cpu().to(dtype=dtype) for m in torch.cat(mids, dim=0).split(1))
    out.append(frames[-1:].to(dtype=dtype))
    return torch.cat(out, dim=0).cpu()


def generic_frame_loop(model_name, frames, clear_cache_after_n_frames, multiplier, return_middle_frame_function,
                       *return_middle_frame_function_args, interpolation_states=None, use_timestep=True,
                       dtype=torch.float32, batch_size=1):
    assert len(frames) >= 2, (f"VFI model {model_name} requires at least 2 frames to work with, "
                              f"only found {frames.shape[0]}.")
    fn, args = return_middle_frame_function, return_middle_frame_function_args
    if type(multiplier) == int:
        return _loop(frames, multiplier, fn, args, interpolation_states, use_timestep, dtype)
    if type(multiplier) == list:
        mults = list(map(int, multiplier))
        mults += [2] * (len(frames) - len(mults) - 1)
        parts = []
        for i in range(len(frames) - 1):
            if mults[i] == 0:
                continue
            part = _loop(frames[i:i + 2], mults[i], fn, args, interpolation_states, use_timestep, dtype)
            parts.append(part if i == len(frames) - 2 else part[:-1])
        return torch.cat(parts)
    raise NotImplementedError(f"multipiler of {type(multiplier)}")
