"""CPU restatement (fp32) of the reference's FILM path (SURVEY.md section 8, row a10).  TEST INFRASTRUCTURE ONLY.

Follows ``vfi_models/film/film_arch.py`` (the model) and ``vfi_models/film/__init__.py`` (the
recursive per-pair schedule and the node loop) of Fannovel16/ComfyUI-Frame-Interpolation @ 26545cc;
every function cites the lines it restates.  As for RIFE, the arithmetic of the reference lives in
PyTorch ATen (``requirements-no-cupy.txt:1``, unpinned; this image: torch 2.11.0) at the call sites
``film_arch.py:717-723`` (grid_sample), ``:598, :611, :751`` (interpolate bilinear), ``:290`` (interpolate
nearest), ``:119, :674`` (avg_pool2d) and ``:786-790`` (conv2d padding='same'); this file calls the same ATen
CPU operators functionally - no ``nn.Module`` and no code from the reference.

Pinning: the reference has no tests or golden vectors for FILM and its checkpoint (a TorchScript file
fetched from a GitHub release) cannot be downloaded here.  ``tools/make_golden_film.py`` therefore runs the
UNMODIFIED ``film_arch.Interpolator`` and the UNMODIFIED ``FILM_VFI.vfi`` (model = ``torch.jit.script`` of the
unmodified Interpolator, saved to a temp file that the stubbed downloader returns) in the build container on
``synthetic_state_dict`` weights and stores their outputs in ``tests/golden/film_*.npz``;
``tests/test_oracle_film.py`` holds this file to them (max abs 1e-6) on every CPU run.

16-bit-faithful mode.  ``interpolator_forward(..., operand="float16" | "bfloat16")`` (and its helpers) evaluate the same
graph in float64 and round to 16 bits (``oracle.rife46.q16``) exactly where the CUDA library stores a 16-bit value, so
that a comparison with the library measures accumulation order only.  With ``operand=None`` (the default) nothing is
rounded and the fp32 graph above runs unchanged, bit for bit.  T is the operand type; where the library stores each
tensor (csrc/film.cu, csrc/film_elem.cu, csrc/streamconv.cu: ``acc + shift``, the activation, then the T store):

| tensor | library | operand mode |
|---|---|---|
| image pyramid | fp32 (``gather_rgb``, ``pool_rgb``) | float64, not rounded |
| ``extract...convs.0.0`` (3 -> 64) | ``conv_rgb``: fp32 weights and bias, output stored in T | unrounded weights, ``round_T(lrelu(y))`` |
| every other conv (streamconv) | weights packed to T, fp32 bias, fp32 accumulation, activation, T store | ``round_T(w)``, bias as is, ``round_T(act(y))`` |
| pooled features, input of sub-level j >= 1 | ``pool16``: fp32 mean of four T values, stored in T | ``round_T(mean)`` |
| up-sampled flow ``2 v`` | ``flow_up``, fp32 | float64 |
| warped features inside the flow estimator | ``warp16``, stored in T | ``round_T(bilinear)`` |
| flow estimator's 1x1 conv output (nf/2 channels) | T (streamconv) | ``round_T`` |
| flow head (nf/2 -> 2) plus the up-sampled flow | ``flow_head``: T inputs, fp32 weights, fp32 output | unrounded weights, float64 |
| aligned features (``warp16``, fscale 0.5) | T | ``round_T`` |
| aligned images and the 0.5-scaled flows | ``misc64``, stored in T | ``round_T(warp(img))``, ``round_T(0.5 flow)`` |
| fusion nearest resize | ``nearest16``, a copy | gather of T values |
| output conv | ``out_rgb``: T inputs, fp32 weights, fp32 output, optional clamp | unrounded weights, float64 |
"""
from __future__ import annotations

import bisect
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from oracle.rife46 import _dt, q16

# Interpolator.__init__ defaults -- film_arch.py:377-386
PYRAMID_LEVELS = 7
FUSION_PYRAMID_LEVELS = 5
SPECIALIZED_LEVELS = 3
SUB_LEVELS = 4
FILTERS = 64
FLOW_CONVS = (3, 3, 3, 3)
FLOW_FILTERS = (32, 64, 128, 256)
LRELU_SLOPE = 0.2  # film_arch.py:797


def _channels_at_level(level: int, filters: int = FILTERS) -> int:
    """film_arch.py:211-216 (get_channels_at_level)."""
    return (sum(filters << i for i in range(level)) + 3 + 2) * 2


def state_dict_spec() -> List[Tuple[str, Tuple[int, ...]]]:
    """Names and shapes of ``Interpolator().state_dict()`` in the reference's order (82 tensors, 34,436,667 values).

    Module construction: SubTreeExtractor film_arch.py:91-100, PyramidFlowEstimator :550-565 (+FlowEstimator
    :515-528), Fusion :222-256; registration order in Interpolator.__init__ :391-393 is extract, predict_flow
    (``_predictor`` before ``_predictors``), fuse (``output_conv`` before ``convs``).  ``conv()`` with an
    activation is ``Sequential(Conv2d, LeakyReLU)`` (hence the extra ``.0``), without one a bare Conv2d (:784-798).
    """
    spec: List[Tuple[str, Tuple[int, ...]]] = []

    def add(name: str, cout: int, cin: int, k: int, seq: bool):
        base = name + (".0" if seq else "")
        spec.append((base + ".weight", (cout, cin, k, k)))
        spec.append((base + ".bias", (cout,)))

    cin = 3
    for i in range(SUB_LEVELS):
        c = FILTERS << i
        add(f"extract.extract_sublevels.convs.{i}.0", c, cin, 3, True)
        add(f"extract.extract_sublevels.convs.{i}.1", c, c, 3, True)
        cin = c

    def flow_estimator(prefix: str, cin: int, num_convs: int, nf: int):
        for j in range(num_convs):
            add(f"{prefix}._convs.{j}", nf, cin, 3, True)
            cin = nf
        add(f"{prefix}._convs.{num_convs}", nf // 2, cin, 1, True)
        add(f"{prefix}._convs.{num_convs + 1}", 2, nf // 2, 1, False)

    in_ch = []
    cin = FILTERS << 1
    for i in range(len(FLOW_CONVS)):
        in_ch.append(cin)
        cin += FILTERS << (i + 2)
    # predictors[-1] is `_predictor`, predictors[:-1][::-1] are `_predictors.{0,1,2}` (levels 2, 1, 0)
    flow_estimator("predict_flow._predictor", in_ch[3], FLOW_CONVS[3], FLOW_FILTERS[3])
    for k, i in enumerate((2, 1, 0)):
        flow_estimator(f"predict_flow._predictors.{k}", in_ch[i], FLOW_CONVS[i], FLOW_FILTERS[i])

    add("fuse.output_conv", 3, FILTERS, 1, False)
    cin = _channels_at_level(SUB_LEVELS)
    increase = 0
    for k, i in enumerate(range(SUB_LEVELS)[::-1]):
        nf = (FILTERS << i) if i < SPECIALIZED_LEVELS else (FILTERS << SPECIALIZED_LEVELS)
        add(f"fuse.convs.{k}.0", nf, cin, 2, False)
        add(f"fuse.convs.{k}.1", nf, cin + (increase or nf), 3, True)
        add(f"fuse.convs.{k}.2", nf, nf, 3, True)
        cin = nf
        increase = _channels_at_level(i) - nf // 2
    return spec


def synthetic_state_dict(seed: int = 0, flow_gain: float = 1.0) -> Dict[str, torch.Tensor]:
    """Seeded stand-in for ``film_net_fp32.pt`` (no weights ship with the reference, no network).

    Variance-preserving uniform weights (LeakyReLU(0.2) gain) so that activations stay O(1) through the 20-odd
    conv layers, the flow heads scaled so that each pyramid level contributes a residual of a fraction of a pixel
    (``flow_gain`` scales it; the coarse levels are doubled on the way up, so full-resolution flows reach tens of
    pixels), and an output conv centred on 0.5 so the image exercises the final clamp on both sides.
    """
    g = torch.Generator().manual_seed(1000 + seed)
    sd: Dict[str, torch.Tensor] = {}
    for name, shape in state_dict_spec():
        if name.endswith(".bias"):
            v = (torch.rand(shape, generator=g) * 2 - 1) * 0.05
            if name == "fuse.output_conv.bias":
                v = v + 0.5
        else:
            fan_in = shape[1] * shape[2] * shape[3]
            a = (6.0 / ((1 + LRELU_SLOPE ** 2) * fan_in)) ** 0.5
            v = (torch.rand(shape, generator=g) * 2 - 1) * a
            if "_convs.4.weight" in name:      # flow head (no activation): residual flow in pixels
                v = v * (0.35 * flow_gain)
            if name == "fuse.output_conv.weight":
                v = v * 0.6
        sd[name] = v.float()
    return sd


def synthetic_clip(n: int, h: int, w: int, seed: int = 1234) -> torch.Tensor:
    """Smooth moving content [n, h, w, 3] in [0, 1]: low-frequency noise translated by (2, 1) px per frame + 2 % noise
    (the generator SURVEY.md section 8d describes for the synthetic clips)."""
    g = torch.Generator().manual_seed(seed)
    base = torch.rand(1, 3, (h + 2 * n) // 16 + 3, (w + 4 * n) // 16 + 3, generator=g)
    big = F.interpolate(base, size=(h + 2 * n, w + 4 * n), mode="bilinear", align_corners=False)[0]
    frames = []
    for i in range(n):
        fr = big[:, i:i + h, 2 * i:2 * i + w]
        frames.append((fr + 0.02 * torch.rand(fr.shape, generator=g)).clamp(0, 1))
    return torch.stack(frames).permute(0, 2, 3, 1).contiguous()


# ------------------------------------------------------------------------------------------------- model
def _conv(sd, name: str, x: torch.Tensor, act: bool, dt=None, packed: bool = True) -> torch.Tensor:
    """film_arch.py:784-798: Conv2d(padding='same') [+ LeakyReLU(0.2)].  For the even (2x2) kernels 'same' pads
    0 rows/columns before and 1 after (ATen conv padding='same': total k-1, the extra one on the right/bottom).
    With a 16-bit type ``dt``: float64, and for a ``packed`` (streamconv) layer the weight and the stored output rounded
    to ``dt``; the CUDA-core layers (``packed=False``) keep fp32 weights and an fp32 output."""
    base = name + (".0" if act else "")
    if dt is None:
        y = F.conv2d(x, sd[base + ".weight"], sd[base + ".bias"], padding="same")
        return F.leaky_relu(y, LRELU_SLOPE) if act else y
    w = sd[base + ".weight"]
    y = F.conv2d(x, q16(w, dt).double() if packed else w.double(), sd[base + ".bias"].double(), padding="same")
    return F.leaky_relu(y, LRELU_SLOPE) if act else y


def build_image_pyramid(image: torch.Tensor, levels: int) -> List[torch.Tensor]:
    """film_arch.py:655-674."""
    pyr = []
    for i in range(levels):
        pyr.append(image)
        if i < levels - 1:
            image = F.avg_pool2d(image, 2, 2)
    return pyr


def sub_tree(sd, image: torch.Tensor, n: int, operand: Optional[str] = None) -> List[torch.Tensor]:
    """SubTreeExtractor.forward, film_arch.py:102-121: all four conv pairs always run; pooling stops after n-1.
    ``operand``: see the module docstring (every conv output and every pooled tensor is stored in T)."""
    dt = _dt(operand)
    head = image
    pyr = []
    for i in range(SUB_LEVELS):
        head = q16(_conv(sd, f"extract.extract_sublevels.convs.{i}.0", head, True, dt, packed=i > 0), dt)
        head = q16(_conv(sd, f"extract.extract_sublevels.convs.{i}.1", head, True, dt), dt)
        pyr.append(head)
        if i < n - 1:
            head = q16(F.avg_pool2d(head, kernel_size=2, stride=2), dt)
    return pyr


def extract(sd, image_pyramid: List[torch.Tensor], operand: Optional[str] = None) -> List[torch.Tensor]:
    """FeatureExtractor.forward, film_arch.py:133-163 (cascaded feature pyramid)."""
    L = len(image_pyramid)
    subs = [sub_tree(sd, image_pyramid[i], min(L - i, SUB_LEVELS), operand) for i in range(L)]
    out = []
    for i in range(L):
        f = subs[i][0]
        for j in range(1, SUB_LEVELS):
            if j <= i:
                f = torch.cat([f, subs[i - j][j]], dim=1)
        out.append(f)
    return out


def warp(image: torch.Tensor, flow: torch.Tensor) -> torch.Tensor:
    """film_arch.py:677-724.  The normalisation there reduces to sampling ``image`` at pixel (x + flow_x, y + flow_y)
    with bilinear weights and border clamping (grid_sample align_corners=False, padding_mode='border'); restated with
    the same operator order so the fp32 rounding matches."""
    fl = -flow.flip(1)
    H, W = fl.shape[2], fl.shape[3]
    ls1 = 1 - 1 / W
    ls2 = 1 - 1 / H
    nf = fl.permute(0, 2, 3, 1) / torch.tensor([H * .5, W * .5], dtype=fl.dtype, device=fl.device)[None, None, None]
    grid = torch.stack([
        torch.linspace(-ls1, ls1, W, dtype=fl.dtype, device=fl.device)[None, None, :] - nf[..., 1],
        torch.linspace(-ls2, ls2, H, dtype=fl.dtype, device=fl.device)[None, :, None] - nf[..., 0],
    ], dim=3)
    out = F.grid_sample(image, grid, mode="bilinear", padding_mode="border", align_corners=False)
    return out.reshape(image.shape)


def flow_estimator(sd, prefix: str, num_convs: int, a: torch.Tensor, b: torch.Tensor,
                   operand: Optional[str] = None) -> torch.Tensor:
    """FlowEstimator.forward, film_arch.py:530-543.  ``operand``: the 3x3 and 1x1 conv outputs stored in T, the head
    (``flow_head``) with fp32 weights and an unrounded output."""
    dt = _dt(operand)
    net = torch.cat([a, b], dim=1)
    for j in range(num_convs + 1):
        net = q16(_conv(sd, f"{prefix}._convs.{j}", net, True, dt), dt)
    return _conv(sd, f"{prefix}._convs.{num_convs + 1}", net, False, dt, packed=False)


def predict_flow(sd, pa: List[torch.Tensor], pb: List[torch.Tensor], operand: Optional[str] = None) -> List[torch.Tensor]:
    """PyramidFlowEstimator.forward, film_arch.py:567-616: residual flow pyramid, fine to coarse.  ``operand``: the warped
    features are stored in T; the flows stay unrounded."""
    dt = _dt(operand)
    levels = len(pa)
    n_spec = len(FLOW_CONVS) - 1  # len(self._predictors)
    v = flow_estimator(sd, "predict_flow._predictor", FLOW_CONVS[3], pa[-1], pb[-1], operand)
    residuals = [v]
    for i in range(levels - 2, n_spec - 1, -1):
        v = F.interpolate(2 * v, size=pa[i].shape[2:4], mode="bilinear")
        warped = q16(warp(pb[i], v), dt)
        r = flow_estimator(sd, "predict_flow._predictor", FLOW_CONVS[3], pa[i], warped, operand)
        residuals.insert(0, r)
        v = r + v
    for k in range(n_spec):
        i = n_spec - 1 - k
        v = F.interpolate(2 * v, size=pa[i].shape[2:4], mode="bilinear")
        warped = q16(warp(pb[i], v), dt)
        r = flow_estimator(sd, f"predict_flow._predictors.{k}", FLOW_CONVS[i], pa[i], warped, operand)
        residuals.insert(0, r)
        v = r + v
    return residuals


def flow_pyramid_synthesis(residuals: List[torch.Tensor]) -> List[torch.Tensor]:
    """film_arch.py:745-755."""
    flow = residuals[-1]
    pyr = [flow]
    for r in residuals[:-1][::-1]:
        flow = F.interpolate(2 * flow, size=r.shape[2:4], mode="bilinear")
        flow = r + flow
        pyr.insert(0, flow)
    return pyr


def fuse(sd, pyramid: List[torch.Tensor], operand: Optional[str] = None) -> torch.Tensor:
    """Fusion.forward, film_arch.py:258-296.  ``operand``: every conv output but the output conv's stored in T (the
    nearest resize copies T values)."""
    dt = _dt(operand)
    net = pyramid[-1]
    n = SUB_LEVELS
    for k in range(n):
        i = n - 1 - k
        net = F.interpolate(net, size=pyramid[i].shape[2:4], mode="nearest")
        net = q16(_conv(sd, f"fuse.convs.{k}.0", net, False, dt), dt)
        net = torch.cat([pyramid[i], net], dim=1)
        net = q16(_conv(sd, f"fuse.convs.{k}.1", net, True, dt), dt)
        net = q16(_conv(sd, f"fuse.convs.{k}.2", net, True, dt), dt)
    return _conv(sd, "fuse.output_conv", net, False, dt, packed=False)


def interpolator_forward(sd, x0: torch.Tensor, x1: torch.Tensor, batch_dt: torch.Tensor,
                         debug: Optional[dict] = None, operand: Optional[str] = None) -> torch.Tensor:
    """Interpolator.forward / debug_forward, film_arch.py:401-459.  x0, x1: [B,3,H,W] fp32, H and W multiples of
    64 are NOT required by the reference (the node feeds frames as they are); ``batch_dt`` only fixes the batch size:
    the network always predicts the midpoint (:424-426).  ``operand``: see the module docstring; ``debug`` then also
    receives ``forward_flow_levels`` / ``backward_flow_levels``, the flows of all seven levels."""
    dt = _dt(operand)
    with torch.no_grad():
        if dt is not None:
            x0, x1 = x0.double(), x1.double()
        ip = [build_image_pyramid(x0, PYRAMID_LEVELS), build_image_pyramid(x1, PYRAMID_LEVELS)]
        fp = [extract(sd, ip[0], operand), extract(sd, ip[1], operand)]
        fwd_res = predict_flow(sd, fp[0], fp[1], operand)
        bwd_res = predict_flow(sd, fp[1], fp[0], operand)
        fwd_all = flow_pyramid_synthesis(fwd_res)
        bwd_all = flow_pyramid_synthesis(bwd_res)
        fwd_pyr = fwd_all[:FUSION_PYRAMID_LEVELS]
        bwd_pyr = bwd_all[:FUSION_PYRAMID_LEVELS]
        mid = torch.full_like(batch_dt, .5)
        bwd = [f * mid[:, 0] for f in bwd_pyr]          # multiply_pyramid, :727-742 (broadcast over the LAST axis
        fwd = [f * (1 - mid[:, 0]) for f in fwd_pyr]    # as written there; exact for batch 1 / equal scalars)
        to_warp = [[torch.cat([ip[k][l], fp[k][l]], dim=1) for l in range(FUSION_PYRAMID_LEVELS)] for k in (0, 1)]
        fw = [q16(warp(a, f), dt) for a, f in zip(to_warp[0], bwd)]
        bw = [q16(warp(a, f), dt) for a, f in zip(to_warp[1], fwd)]
        aligned = [torch.cat([a, b, q16(c, dt), q16(d, dt)], dim=1) for a, b, c, d in zip(fw, bw, bwd, fwd)]
        if debug is not None:
            debug.update(feature_pyramids=fp, forward_residual=fwd_res, backward_residual=bwd_res,
                         forward_flow=fwd_pyr, backward_flow=bwd_pyr, aligned=aligned,
                         forward_flow_levels=fwd_all, backward_flow_levels=bwd_all)
        return fuse(sd, aligned, operand)


# ------------------------------------------------------------------------------------------------- node
def inference_order(inter_frames: int) -> List[Tuple[int, int, int]]:
    """The bisection schedule of ``inference`` (film/__init__.py:12-42) as a list of (left index, right index,
    new index) into the final sequence 0..inter_frames+1: at every step the (segment, remaining position) pair whose
    position is closest to the middle of its segment is generated from the segment's two ends, always at dt 0.5 in
    effect (the model ignores dt)."""
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
        bisect.insort_left(idxes, remains[step])
        del remains[step]
    return order


def inference(sd, f0: torch.Tensor, f1: torch.Tensor, inter_frames: int) -> List[torch.Tensor]:
    """film/__init__.py:12-42 incl. its final ``flip(0)`` of every (batch-1) tensor, which is the identity."""
    res = {0: f0, inter_frames + 1: f1}
    for lo, hi, new in inference_order(inter_frames):
        dt = f0.new_full((1, 1), 0.5)
        res[new] = interpolator_forward(sd, res[lo], res[hi], dt).clamp(0, 1).float()
    return [res[i] for i in range(inter_frames + 2)]


def film_vfi(sd, frames: torch.Tensor, multiplier=2, states: Optional[Tuple[Sequence[int], bool]] = None
             ) -> torch.Tensor:
    """FILM_VFI.vfi, film/__init__.py:63-113.  frames [N,H,W,C>=3] fp32 -> [M,H,W,3] fp32.  A skipped pair is
    DROPPED with its first frame (``continue`` at :85-86, unlike RIFE); the multiplier list is padded with 2s
    (:81-83); the last frame is always appended (:104)."""
    x = frames[..., :3].permute(0, 3, 1, 2)  # preprocess_frames, vfi_utils.py:139-140
    n = x.shape[0]
    if isinstance(multiplier, int):
        mults = [multiplier] * n
    else:
        mults = list(map(int, multiplier))
        mults += [2] * (n - len(mults) - 1)
    out = []
    for i in range(n - 1):
        if states is not None and is_frame_skipped(states, i):
            continue
        res = inference(sd, x[i:i + 1].float(), x[i + 1:i + 2].float(), mults[i] - 1)
        out.extend(r.to(torch.float32) for r in res[:-1])
    out.append(x[-1:].to(torch.float32))
    return torch.cat(out, dim=0).permute(0, 2, 3, 1)  # postprocess_frames, vfi_utils.py:142-143


def is_frame_skipped(states: Tuple[Sequence[int], bool], idx: int) -> bool:
    """InterpolationStateList.is_frame_skipped, vfi_utils.py:55-57."""
    frame_indices, is_skip_list = states
    in_list = idx in frame_indices
    return (is_skip_list and in_list) or (not is_skip_list and not in_list)
