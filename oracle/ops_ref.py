"""CPU restatement of the reference's custom CUDA ops (`vfi_models/ops/cupy_ops`).  TEST INFRASTRUCTURE ONLY.

cupy is not installed in this image (and the reference's taichi backend does not import, SURVEY.md F6), so the
reference kernels cannot be launched as the reference launches them.  Pinning: `oracle/ref_ops.py` specialises the reference's
own kernel strings with the reference's own pre-processor and runs them on the CPU (g++ through tests/host_emu);
`tests/test_ops_ref_pinned.py` holds `softsplat_sum` / `softsplat` / `costvol_l1` / `correlation_dot` / `sepconv` below to
those outputs.  Each function below follows the
CUDA-C source string of the reference kernel line by line (cited), in fp32 on NCHW tensors like the reference,
and is cross-checked in tests/test_ops_ref.py against independent formulations (grid_sample adjoint for the splat,
unfold-based volumes, explicit double loops on tiny inputs).
"""
import torch
import torch.nn.functional as F


def softsplat_sum(ten_in: torch.Tensor, ten_flow: torch.Tensor) -> torch.Tensor:
    """softsplat_out - cupy_ops/softsplat.py:140-192 (summation splatting).

    Each source pixel (n,c,y,x) adds in*w to its four bilinear neighbours of (x+fx, y+fy); targets outside the image
    are dropped; a non-finite flow drops the pixel.  The reference uses atomicAdd (order nondeterministic); here the
    sum is accumulated with index_add_ in float64 and rounded once, so agreement with any summation order is ~1 ulp
    of the partial sums.  The corner weights are computed in the flow's dtype and the result is returned in the input's
    (fp32 like the reference, or float64 throughout), on the inputs' device."""
    n, c, h, w = ten_in.shape
    dt, dev = ten_flow.dtype, ten_flow.device
    out = torch.zeros(n, c, h * w, dtype=torch.float64, device=dev)
    ys, xs = torch.meshgrid(torch.arange(h, dtype=dt, device=dev), torch.arange(w, dtype=dt, device=dev), indexing="ij")
    for b in range(n):
        fx = xs + ten_flow[b, 0]
        fy = ys + ten_flow[b, 1]
        ok = torch.isfinite(fx) & torch.isfinite(fy)
        fx = torch.where(ok, fx, torch.zeros_like(fx))
        fy = torch.where(ok, fy, torch.zeros_like(fy))
        x0 = torch.floor(fx)
        y0 = torch.floor(fy)
        src = ten_in[b].reshape(c, -1).double()
        for dx, dy in ((0, 0), (1, 0), (0, 1), (1, 1)):
            tx, ty = x0 + dx, y0 + dy
            # weight of the corner = product of distances to the OPPOSITE corner (:166-169), computed in fp32
            wx = ((x0 + 1) - fx) if dx == 0 else (fx - x0)
            wy = ((y0 + 1) - fy) if dy == 0 else (fy - y0)
            wgt = (wx * wy)
            inside = ok & (tx >= 0) & (tx < w) & (ty >= 0) & (ty < h)
            idx = (ty.clamp(0, h - 1) * w + tx.clamp(0, w - 1)).long().reshape(-1)
            contrib = (src.to(dt) * wgt.reshape(1, -1)).double() * inside.reshape(1, -1)
            out[b].index_add_(1, idx, contrib)
    return out.reshape(n, c, h, w).to(ten_in.dtype)


def softsplat(ten_in, ten_flow, ten_metric, mode: str):
    """softsplat() wrapper - cupy_ops/softsplat.py:382-435: modes sum / avg / linear / soft with the -addeps (default),
    -zeroeps, -clipeps normalisation variants."""
    base = mode.split("-")[0]
    assert base in ("sum", "avg", "linear", "soft")
    if base == "avg":
        ten_in = torch.cat([ten_in, ten_in.new_ones(ten_in.shape[0], 1, *ten_in.shape[2:])], 1)
    elif base == "linear":
        ten_in = torch.cat([ten_in * ten_metric, ten_metric], 1)
    elif base == "soft":
        ten_in = torch.cat([ten_in * ten_metric.exp(), ten_metric.exp()], 1)
    out = softsplat_sum(ten_in, ten_flow)
    if base in ("avg", "linear", "soft"):
        norm = out[:, -1:]
        variant = mode.split("-")[1] if "-" in mode else "addeps"
        if variant == "addeps":
            norm = norm + 0.0000001
        elif variant == "zeroeps":
            norm = norm.clone()
            norm[norm == 0.0] = 1.0
        elif variant == "clipeps":
            norm = norm.clip(0.0000001, None)
        out = out[:, :-1] / norm
    return out


def costvol_l1(one: torch.Tensor, two: torch.Tensor) -> torch.Tensor:
    """costvol_out - cupy_ops/costvol.py:4-43: out[n, k, y, x] = mean_c |one[c,y,x] - two[c,y+dy,x+dx]| for the 9x9
    displacements (dy outer, dx inner, -4..4); a displaced position outside the image gives mean_c |one[c,y,x]|."""
    n, c, h, w = one.shape
    out = torch.empty(n, 81, h, w)
    k = 0
    for dy in range(-4, 5):
        for dx in range(-4, 5):
            shifted = torch.zeros_like(two)
            ys0, ys1 = max(0, -dy), min(h, h - dy)
            xs0, xs1 = max(0, -dx), min(w, w - dx)
            if ys1 > ys0 and xs1 > xs0:
                shifted[:, :, ys0:ys1, xs0:xs1] = two[:, :, ys0 + dy:ys1 + dy, xs0 + dx:xs1 + dx]
            # outside: shifted == 0 so |one - 0| = |one|, exactly the reference's else-branch
            out[:, k] = (one - shifted).abs().sum(1) / c
            k += 1
    return out


def correlation_dot(first: torch.Tensor, second: torch.Tensor) -> torch.Tensor:
    """FunctionCorrelation - cupy_ops/correlation.py:4-99 (+ wrapper :231-296): both inputs zero padded by 4
    (rearrange kernel), out[n, k, y, x] = mean_c first[c,y,x] * second[c, y+s2p, x+s2o], k = (s2p+4)*9 + (s2o+4)."""
    n, c, h, w = first.shape
    sp = F.pad(second, (4, 4, 4, 4))
    out = torch.empty(n, 81, h, w)
    for k in range(81):
        s2o, s2p = k % 9 - 4, k // 9 - 4
        out[:, k] = (first * sp[:, :, 4 + s2p:4 + s2p + h, 4 + s2o:4 + s2o + w]).sum(1) / c
    return out


def sepconv(ten_in: torch.Tensor, ver: torch.Tensor, hor: torch.Tensor) -> torch.Tensor:
    """sepconv_out - cupy_ops/sepconv.py:86-117: out[n,c,y,x] = sum_fy sum_fx in[n,c,y+fy,x+fx]*ver[n,fy,y,x]*hor[n,fx,y,x]
    (`in` is already padded by K-1), accumulated with Kahan summation in that loop order.  Here: float64 sum of the
    fp32 products (Kahan's purpose is an accurately rounded fp32 sum, so the two agree to ~1 ulp)."""
    n, c, hp, wp = ten_in.shape
    kv, kh = ver.shape[1], hor.shape[1]
    h, w = ver.shape[2], ver.shape[3]
    assert hp == h + kv - 1 and wp == w + kh - 1
    out = torch.zeros(n, c, h, w, dtype=torch.float64)
    for fy in range(kv):
        for fx in range(kh):
            prod = ten_in[:, :, fy:fy + h, fx:fx + w] * ver[:, fy:fy + 1] * hor[:, fx:fx + 1]
            out += prod.double()
    return out.float()


def adacof(inp: torch.Tensor, weight: torch.Tensor, off_i: torch.Tensor, off_j: torch.Tensor, dilation: int) -> torch.Tensor:
    """kernel_AdaCoF_updateOutput - cupy_ops/adacof.py:5-62: for every tap (k, l) the input is sampled at
    (i + k d + alpha, j + l d + beta) with A = (int) alpha TRUNCATED toward zero, the four tap indices clamped to the
    image and the (unclamped, possibly negative) fractions alpha - A, beta - B as weights."""
    n, c, hin, win = inp.shape
    f = int(round(weight.shape[1] ** 0.5))
    ho, wo = weight.shape[2], weight.shape[3]
    ii = torch.arange(ho).view(1, ho, 1)
    jj = torch.arange(wo).view(1, 1, wo)
    nn = torch.arange(n).view(n, 1, 1)
    out = torch.zeros(n, c, ho, wo, dtype=torch.float64)
    for k in range(f):
        for l in range(f):
            t = k * f + l
            w, al, be = weight[:, t], off_i[:, t], off_j[:, t]
            a_, b_ = al.to(torch.int32).long(), be.to(torch.int32).long()   # C cast: truncation toward zero
            y0 = (ii + k * dilation + a_).clamp(0, hin - 1)
            y1 = (ii + k * dilation + a_ + 1).clamp(0, hin - 1)
            x0 = (jj + l * dilation + b_).clamp(0, win - 1)
            x1 = (jj + l * dilation + b_ + 1).clamp(0, win - 1)
            fa, fb = (al - a_.float()), (be - b_.float())
            g = lambda y, x: inp[nn, :, y, x].permute(0, 3, 1, 2)   # noqa: E731  -> [n, c, ho, wo]
            val = (g(y0, x0) * ((1 - fa) * (1 - fb)).unsqueeze(1) + g(y1, x0) * (fa * (1 - fb)).unsqueeze(1) +
                   g(y0, x1) * ((1 - fa) * fb).unsqueeze(1) + g(y1, x1) * (fa * fb).unsqueeze(1))
            out += (w.unsqueeze(1) * val).double()
    return out.float()


def edt_pass(data: torch.Tensor, diam2: float) -> torch.Tensor:
    """kernel_dt - cupy_ops/batch_edt.py:9-41: out[b,i,j] = min(diam2, min_j' data[b,i,j'] + (j - j')^2)."""
    w = data.shape[-1]
    j = torch.arange(w, dtype=torch.float32)
    cost = data.unsqueeze(-2) + (j.view(-1, 1) - j.view(1, -1)) ** 2      # [..., j, j']
    return torch.minimum(cost.min(-1).values, torch.tensor(float(diam2)))


def batch_edt(img: torch.Tensor) -> torch.Tensor:
    """batch_edt - cupy_ops/batch_edt.py:46-117 (the cupy branch): two kernel_dt passes around a transpose, then sqrt."""
    expand = img.dim() == 4
    if expand:
        img = img.squeeze(1)
    bs, h, w = img.shape
    diam2 = h ** 2 + w ** 2
    data = (1 - img.float()) * diam2
    inter = edt_pass(data, diam2).permute(0, 2, 1).contiguous()
    ans = edt_pass(inter, diam2).permute(0, 2, 1).sqrt().to(img.dtype)
    return ans.unsqueeze(1) if expand else ans
