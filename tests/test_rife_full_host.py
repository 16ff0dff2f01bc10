"""The WHOLE RIFE path of the library on the CPU: csrc/rife46.cu (vfi_create / vfi_rife_load / vfi_rife46_forward: weight
repacking, the per-block schedule with its implicit full-resolution flow, the C ABI), csrc/elementwise.cu (prep / front /
final kernels with their 3-D launch geometry) and csrc/tapconv.cu's plan + CUDA-core checker kernel, compiled for the host
(tests/host_emu/cuda_shim_block.h: every thread of every block a fiber) and compared with the unmodified reference IFNet's
output (tests/golden).  The wgmma kernel is covered by the GPU tests (tests/test_gpu_layers.py: wgmma vs this checker)."""
import ctypes as C
import math
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden import cases, make_inputs  # noqa: E402
from oracle import rife46 as O  # noqa: E402
import rife16_util as U  # noqa: E402

CUDA_INC = "/usr/local/cuda/include"


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not (shutil.which("g++") and os.path.exists(os.path.join(CUDA_INC, "cuda_fp16.h"))):
        pytest.skip("g++ / CUDA headers not available")
    so = str(tmp_path_factory.mktemp("emu") / "librifefull.so")
    src = os.path.join(ROOT, "tests", "host_emu", "rife_full_emu.cpp")
    r = subprocess.run(["g++", "-O2", "-std=c++20", "-shared", "-fPIC", "-pthread", "-I" + CUDA_INC, "-o", so, src] + os.environ.get("VFI_EMU_CXXFLAGS", "").split(),
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(so)
    L.vfi_last_error.restype = C.c_char_p
    return L


def _engine_names(arch):
    import __graft_entry__ as ge
    ge.load_package()
    from cfi_b200.engine import ARCH_CODE, state_dict_names
    return state_dict_names(arch), ARCH_CODE[arch]


def _run(emu, arch, sd, fr, ts, sf, operand):
    """One emulated vfi_rife46_forward of the tasks (0, 1, ts[i]): (frames [B,h,w,3], flow [B,Hp,Wp,4], mask [B,Hp,Wp])."""
    names, code = _engine_names(arch)
    hold = [sd[n].contiguous().float() for n in names]
    ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
    numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
    ctx = C.c_void_p()
    assert emu.vfi_create(0, C.byref(ctx)) == 0, emu.vfi_last_error()
    assert emu.vfi_rife_load(ctx, code, ptrs, numel, len(hold), 0 if operand == "float16" else 1) == 0, emu.vfi_last_error()
    fr = fr.contiguous()
    n, h, w, c = fr.shape
    b = len(ts)
    t = np.asarray(ts, np.float32)
    f0, f1 = np.zeros(b, np.int32), np.ones(b, np.int32)
    vp = lambda x: x.ctypes.data_as(C.c_void_p)   # noqa: E731
    out = torch.zeros(b, h, w, 3)
    assert emu.vfi_rife46_forward(ctx, C.c_void_p(fr.data_ptr()), n, h, w, c, vp(f0), vp(f1), vp(t), b, C.c_float(sf),
                                  C.c_void_p(out.data_ptr()), None) == 0, emu.vfi_last_error()
    hp, wp = C.c_int(), C.c_int()
    assert emu.vfi_rife46_debug_state(ctx, None, None, b, C.byref(hp), C.byref(wp)) == 0, emu.vfi_last_error()
    flow, mask = torch.zeros(b, hp.value, wp.value, 4), torch.zeros(b, hp.value, wp.value)
    assert emu.vfi_rife46_debug_state(ctx, C.c_void_p(flow.data_ptr()), C.c_void_p(mask.data_ptr()), b, C.byref(hp),
                                      C.byref(wp)) == 0, emu.vfi_last_error()
    assert emu.vfi_destroy(ctx) == 0
    return out, flow, mask


def _check_faithful(emu, label, arch, sd, fr, ts, sf, operand):
    """The emulated path against the 16-bit-faithful float64 oracle, per pixel (tests/rife16_util.py)."""
    got = _run(emu, arch, sd, fr, ts, sf, operand)
    want = U.oracle(arch, sd, fr, [0] * len(ts), [1] * len(ts), ts, sf, operand)
    lines, fails = U.compare(f"{label} {operand}", got, want, fr.shape[1], fr.shape[2], U.tol(label, operand))
    print("\n".join(lines))
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("operand", ["float16", "bfloat16"])
@pytest.mark.parametrize("arch,sf,h,w", [pytest.param(*c, id=U.case_id(*c)) for c in U.cases()])
def test_rife_whole_path_on_host_matches_faithful_oracle(emu, arch, sf, h, w, operand):
    """Odd sizes, a thin strip, t near 0 and 1 and every scale_factor: frames, full-resolution flow and mask of the
    emulated library against the 16-bit-faithful oracle, over the whole plane and over its border band."""
    sd, fr = U.inputs(arch, h, w)
    _check_faithful(emu, U.case_id(arch, sf, h, w), arch, sd, fr, list(U.TIMESTEPS), sf, operand)


@pytest.mark.parametrize("name", ["ifnet_64x64_gain4", "ifnet47_64x128_gain3", "ifnet417_64x128_gain3",
                                  "ifnet426_128x128_gain3", "ifnet_64x64_sf2", "ifnet_64x64_sf4", "ifnet47_64x64_sf2",
                                  "ifnet47_64x64_sf4", "ifnet417_64x64_sf2", "ifnet426_64x64_sf2",
                                  "ifnet426_64x64_sf4", "ifnet_40x100_sf2", "ifnet426_40x100_sf4"])
def test_rife_whole_path_on_host_matches_reference(emu, name):
    cfg = cases()[name]
    arch = cfg.get("arch", "4.6")
    ref = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))["out"]).permute(0, 2, 3, 1)
    sd = O.synthetic_state_dict(cfg["seed"], cfg["gain"], arch=arch)
    names, code = _engine_names(arch)
    hold = [sd[n].contiguous().float() for n in names]
    ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
    numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
    ctx = C.c_void_p()
    assert emu.vfi_create(0, C.byref(ctx)) == 0, emu.vfi_last_error()
    assert emu.vfi_rife_load(ctx, code, ptrs, numel, len(hold), 0) == 0, emu.vfi_last_error()
    fr = make_inputs(cfg).contiguous()
    n, h, w, c = fr.shape
    ts = np.asarray(cfg["ts"], dtype=np.float32)
    f0 = np.zeros(len(ts), dtype=np.int32)
    f1 = np.ones(len(ts), dtype=np.int32)
    out = torch.zeros(len(ts), h, w, 3)
    rc = emu.vfi_rife46_forward(ctx, C.c_void_p(fr.data_ptr()), n, h, w, c, f0.ctypes.data_as(C.c_void_p),
                                f1.ctypes.data_as(C.c_void_p), ts.ctypes.data_as(C.c_void_p), len(ts),
                                C.c_float(cfg.get("scale_factor", 1.0)),
                                C.c_void_p(out.data_ptr()), None)
    assert rc == 0, emu.vfi_last_error()
    emu.vfi_launch_count.restype = C.c_int64
    launches = emu.vfi_launch_count(ctx)
    assert emu.vfi_destroy(ctx) == 0
    want = ref.clamp(0, 1)   # the library returns the node's clamped frame (rife/__init__.py:207)
    mse = float(((out.double() - want.double()) ** 2).mean())
    psnr = 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)
    print(f"host emulation of the whole RIFE {arch} path ({name}): {launches} launches, PSNR {psnr:.2f} dB")
    assert psnr >= 60.0, psnr
    _check_faithful(emu, name, arch, sd, fr, list(cfg["ts"]), cfg.get("scale_factor", 1.0), "float16")


def test_rife_bf16_operands_on_host(emu):
    """node dtype bfloat16 = bf16 conv operands (VFI_OPERAND_BF16): the bf16 instantiations of the element-wise kernels and of
    the checker, same schedule; the bar is the north_star's 50 dB."""
    name = "ifnet_64x64_gain4"
    cfg = cases()[name]
    ref = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))["out"]).permute(0, 2, 3, 1).clamp(0, 1)
    sd = O.synthetic_state_dict(cfg["seed"], cfg["gain"])
    names, code = _engine_names("4.6")
    hold = [sd[n].contiguous().float() for n in names]
    ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
    numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
    ctx = C.c_void_p()
    assert emu.vfi_create(0, C.byref(ctx)) == 0
    assert emu.vfi_rife_load(ctx, code, ptrs, numel, len(hold), 1) == 0, emu.vfi_last_error()
    fr = make_inputs(cfg).contiguous()
    n, h, w, c = fr.shape
    f0, f1, ts = np.zeros(1, np.int32), np.ones(1, np.int32), np.asarray(cfg["ts"], np.float32)
    out = torch.zeros(1, h, w, 3)
    vp = lambda x: x.ctypes.data_as(C.c_void_p)   # noqa: E731
    assert emu.vfi_rife46_forward(ctx, C.c_void_p(fr.data_ptr()), n, h, w, c, vp(f0), vp(f1), vp(ts), 1, C.c_float(1.0),
                                  C.c_void_p(out.data_ptr()), None) == 0, emu.vfi_last_error()
    assert emu.vfi_destroy(ctx) == 0
    mse = float(((out.double() - ref.double()) ** 2).mean())
    psnr = 10 * math.log10(1.0 / mse)
    print(f"host emulation, bf16 operands ({name}): PSNR {psnr:.2f} dB")
    assert psnr >= 50.0, psnr


@pytest.mark.parametrize("name", ["ifnet_64x64_gain4", "ifnet47_64x128_gain3", "ifnet417_64x128_gain3",
                                  "ifnet426_128x128_gain3", "ifnet_64x64_sf2", "ifnet_64x64_sf4", "ifnet47_64x64_sf2",
                                  "ifnet47_64x64_sf4", "ifnet417_64x64_sf2", "ifnet426_64x64_sf2",
                                  "ifnet426_64x64_sf4", "ifnet_40x100_sf2", "ifnet426_40x100_sf4"])
def test_rife_bf16_golden_cases_on_host_match_faithful_oracle(emu, name):
    """The golden cases with bf16 operands against the 16-bit-faithful oracle, per pixel."""
    cfg = cases()[name]
    arch = cfg.get("arch", "4.6")
    sd = O.synthetic_state_dict(cfg["seed"], cfg["gain"], arch=arch)
    _check_faithful(emu, name, arch, sd, make_inputs(cfg), list(cfg["ts"]), cfg.get("scale_factor", 1.0), "bfloat16")


def test_rife_host_pipeline_on_host_matches_reference_node(emu):
    """vfi_rife46_interpolate_host (the H2D / compute / D2H pipeline with its ring of raw frames and output slots) against
    the unmodified reference node's output: multiplier 3, a skipped pair, 4-channel frames (tests/golden/node_m3_skip.npz)."""
    import __graft_entry__ as ge
    ge.load_package()
    import cfi_b200.node as N
    name = "node_m3_skip"
    cfg = cases()[name]
    ref = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))["out"])
    sd = O.synthetic_state_dict(cfg["seed"], cfg["gain"])
    names, code = _engine_names("4.6")
    hold = [sd[n].contiguous().float() for n in names]
    ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
    numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
    ctx = C.c_void_p()
    assert emu.vfi_create(0, C.byref(ctx)) == 0, emu.vfi_last_error()
    assert emu.vfi_rife_load(ctx, code, ptrs, numel, len(hold), 0) == 0, emu.vfi_last_error()
    fr = make_inputs(cfg).contiguous()
    n, h, w, c = fr.shape
    st = N.InterpolationStateList(list(cfg["states"][0]), cfg["states"][1])
    tasks, _ = N.build_tasks(n - 1, cfg["multiplier"], st)
    # output slots exactly as node.RIFE_VFI.vfi lays them out
    per_pair = [0] * (n - 1)
    for p_, _t in tasks:
        per_pair[p_] += 1
    first_slot, slot = [], 0
    for p_ in range(n - 1):
        first_slot.append(slot)
        slot += 1 + per_pair[p_]
    total = slot + 1
    out = torch.zeros(total, h, w, 3)
    seen = [0] * (n - 1)
    f0, f1, ts, slots = [], [], [], []
    for p_, t in tasks:
        seen[p_] += 1
        f0.append(p_); f1.append(p_ + 1); ts.append(t); slots.append(first_slot[p_] + seen[p_])
    a = lambda v, dt: np.ascontiguousarray(np.asarray(v, dtype=dt))   # noqa: E731
    f0a, f1a, tsa, sla = a(f0, np.int32), a(f1, np.int32), a(ts, np.float32), a(slots, np.int32)
    vp = lambda x: x.ctypes.data_as(C.c_void_p)   # noqa: E731
    rc = emu.vfi_rife46_interpolate_host(ctx, C.c_void_p(fr.data_ptr()), n, h, w, c, 0, n, vp(f0a), vp(f1a), vp(tsa), vp(sla), None,
                                         len(ts), C.c_float(1.0), C.c_void_p(out.data_ptr()))
    assert rc == 0, emu.vfi_last_error()
    assert emu.vfi_destroy(ctx) == 0
    out[first_slot + [total - 1]] = fr[..., :3]          # the node copies the pass-through frames itself
    assert out.shape == ref.shape
    mse = float(((out.double() - ref.double()) ** 2).mean())
    psnr = 99.0 if mse == 0 else 10 * math.log10(1.0 / mse)
    print(f"host emulation of the RIFE host pipeline ({name}): PSNR {psnr:.2f} dB")
    assert psnr >= 60.0, psnr


def test_rife_host_pipeline_ring_and_shards_on_host(emu):
    """The host pipeline's bookkeeping on the CPU: more tasks than one internal pass holds (batch 2: ramped pass sizes, the
    ring of uploaded source frames, double-buffered output), out-of-order output slots and a frame shard [frame_lo,
    frame_hi) - every task's frame must equal what the device-level entry point returns for the same (pair, timestep)."""
    names, code = _engine_names("4.6")
    sd = O.synthetic_state_dict(7, 1.0)
    hold = [sd[n].contiguous().float() for n in names]
    ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
    numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
    ctx = C.c_void_p()
    assert emu.vfi_create(0, C.byref(ctx)) == 0, emu.vfi_last_error()
    assert emu.vfi_rife_load(ctx, code, ptrs, numel, len(hold), 0) == 0, emu.vfi_last_error()
    assert emu.vfi_set_batch(ctx, 2) == 0
    n, h, w, c = 7, 40, 56, 3
    fr = O.synthetic_clip(n, h, w, seed=77).contiguous()
    # shard: only frames [1, 6) may be touched; tasks on pairs 1..4, two timesteps on pair 2, slots reversed
    tasks = [(1, 0.5), (2, 0.25), (2, 0.75), (3, 0.5), (4, 0.5)]
    f0 = np.asarray([p for p, _ in tasks], dtype=np.int32)
    f1 = f0 + 1
    ts = np.asarray([t for _, t in tasks], dtype=np.float32)
    slots = np.asarray(list(range(len(tasks)))[::-1], dtype=np.int32)
    vp = lambda x: x.ctypes.data_as(C.c_void_p)   # noqa: E731
    out = torch.zeros(len(tasks), h, w, 3)
    rc = emu.vfi_rife46_interpolate_host(ctx, C.c_void_p(fr.data_ptr()), n, h, w, c, 1, 6, vp(f0), vp(f1), vp(ts), vp(slots), None,
                                         len(tasks), C.c_float(1.0), C.c_void_p(out.data_ptr()))
    assert rc == 0, emu.vfi_last_error()
    for i, (p_, t) in enumerate(tasks):
        one = torch.zeros(1, h, w, 3)
        a0, a1, at = np.asarray([p_], np.int32), np.asarray([p_ + 1], np.int32), np.asarray([t], np.float32)
        assert emu.vfi_rife46_forward(ctx, C.c_void_p(fr.data_ptr()), n, h, w, c, vp(a0), vp(a1), vp(at), 1, C.c_float(1.0),
                                      C.c_void_p(one.data_ptr()), None) == 0, emu.vfi_last_error()
        assert torch.equal(out[slots[i]], one[0]), (i, p_, t)
    # a longer task list with gaps (skipped pairs: their frames are never uploaded), a prepared-frame ring that wraps
    # several times and pinned staging rings of two slots (every caller buffer counts as pageable in the emulation)
    n2 = 12
    fr2 = O.synthetic_clip(n2, h, w, seed=78).contiguous()
    tasks2 = [(0, 0.5), (1, 0.5), (1, 0.25), (4, 0.5), (5, 0.5), (6, 0.75), (9, 0.5), (10, 0.5)]
    g0 = np.asarray([p for p, _ in tasks2], dtype=np.int32)
    g1 = g0 + 1
    gt = np.asarray([t for _, t in tasks2], dtype=np.float32)
    out2 = torch.zeros(len(tasks2), h, w, 3)
    os.environ["VFI_STAGE_SLOTS"] = "2"
    try:
        rc = emu.vfi_rife46_interpolate_host(ctx, C.c_void_p(fr2.data_ptr()), n2, h, w, c, 0, n2, vp(g0), vp(g1), vp(gt), None, None,
                                             len(tasks2), C.c_float(1.0), C.c_void_p(out2.data_ptr()))
    finally:
        del os.environ["VFI_STAGE_SLOTS"]
    assert rc == 0, emu.vfi_last_error()
    # the same with pass-through slots (what the node does): frames 0..11 -> slots 20.., 4-channel source, frame 3 and 8 are
    # referenced by no task, frame 7 has no slot
    fr4 = torch.cat([fr2, torch.full((n2, h, w, 1), 0.25)], -1).contiguous()
    big = torch.full((40, h, w, 3), -1.0)
    fs = np.asarray([20 + i for i in range(n2)], dtype=np.int32)
    fs[7] = -1
    sl2 = np.arange(len(tasks2), dtype=np.int32)
    os.environ["VFI_STAGE_SLOTS"] = "2"
    try:
        rc = emu.vfi_rife46_interpolate_host(ctx, C.c_void_p(fr4.data_ptr()), n2, h, w, 4, 0, n2, vp(g0), vp(g1), vp(gt), vp(sl2),
                                             vp(fs), len(tasks2), C.c_float(1.0), C.c_void_p(big.data_ptr()))
    finally:
        del os.environ["VFI_STAGE_SLOTS"]
    assert rc == 0, emu.vfi_last_error()
    assert torch.equal(big[: len(tasks2)], out2)
    for i in range(n2):
        if i != 7:
            assert torch.equal(big[20 + i], fr2[i]), i
    assert float(big[27].max()) == -1.0 and float(big[len(tasks2):20].max()) == -1.0
    for i, (p_, t) in enumerate(tasks2):
        one = torch.zeros(1, h, w, 3)
        a0, a1, at = np.asarray([p_], np.int32), np.asarray([p_ + 1], np.int32), np.asarray([t], np.float32)
        assert emu.vfi_rife46_forward(ctx, C.c_void_p(fr2.data_ptr()), n2, h, w, c, vp(a0), vp(a1), vp(at), 1, C.c_float(1.0),
                                      C.c_void_p(one.data_ptr()), None) == 0, emu.vfi_last_error()
        assert torch.equal(out2[i], one[0]), (i, p_, t)
    # a task outside the shard is refused
    bad0, bad1 = np.asarray([0], np.int32), np.asarray([1], np.int32)
    rc = emu.vfi_rife46_interpolate_host(ctx, C.c_void_p(fr.data_ptr()), n, h, w, c, 1, 6, vp(bad0), vp(bad1), vp(ts), None, None, 1,
                                         C.c_float(1.0), C.c_void_p(out.data_ptr()))
    assert rc != 0
    assert emu.vfi_destroy(ctx) == 0


@pytest.mark.parametrize("sf", [1.0, 2.0])
def test_rife_flow_state_on_host(emu, sf):
    """vfi_rife46_debug_state: the accumulated full-resolution flow / mask of the last pass (implicit on the product path;
    with scale_factor 2 every level has already been folded into the dense planes) against the oracle's final flow and
    mask, in pixels."""
    sd = O.synthetic_state_dict(11, 3.0)
    names, code = _engine_names("4.6")
    hold = [sd[n].contiguous().float() for n in names]
    ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
    numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
    ctx = C.c_void_p()
    assert emu.vfi_create(0, C.byref(ctx)) == 0
    assert emu.vfi_rife_load(ctx, code, ptrs, numel, len(hold), 0) == 0, emu.vfi_last_error()
    fr = O.synthetic_clip(2, 64, 64, seed=5).contiguous()
    f0, f1, ts = np.zeros(1, np.int32), np.ones(1, np.int32), np.asarray([0.5], np.float32)
    out = torch.zeros(1, 64, 64, 3)
    vp = lambda x: x.ctypes.data_as(C.c_void_p)   # noqa: E731
    assert emu.vfi_rife46_forward(ctx, C.c_void_p(fr.data_ptr()), 2, 64, 64, 3, vp(f0), vp(f1), vp(ts), 1, C.c_float(sf),
                                  C.c_void_p(out.data_ptr()), None) == 0, emu.vfi_last_error()
    hp, wp = C.c_int(), C.c_int()
    flow = torch.zeros(1, 64, 64, 4)
    mask = torch.zeros(1, 64, 64)
    assert emu.vfi_rife46_debug_state(ctx, C.c_void_p(flow.data_ptr()), C.c_void_p(mask.data_ptr()), 1, C.byref(hp),
                                      C.byref(wp)) == 0, emu.vfi_last_error()
    assert (hp.value, wp.value) == (64, 64)
    assert emu.vfi_destroy(ctx) == 0
    taps = {}
    x = fr.permute(0, 3, 1, 2)
    O.ifnet46_forward(sd, x[0:1], x[1:2], torch.tensor([0.5]).view(1, 1, 1, 1), [v / sf for v in (8, 4, 2, 1)], taps)
    want_f, want_m = taps["flow3"].permute(0, 2, 3, 1), taps["mask3"][:, 0]
    assert float(want_f.abs().max()) > 2.0                       # a few pixels of motion
    assert (flow - want_f).abs().max().item() <= 0.05            # fp16 conv operands: hundredths of a pixel
    assert (mask - want_m).abs().max().item() <= 0.05


@pytest.mark.parametrize("operand", ["float16", "bfloat16"])
@pytest.mark.parametrize("arch", ["4.6", "4.26"])
def test_streamed_weight_plans_on_host(emu, arch, operand):
    """vfi_rife46_layer_plan of the loaded library: exactly the layers test_gpu_tapconv_wstream.py expects stream their
    weights (blocks 0-2's ResConvs, block 1's lastconv, 4.26's feature conv of blocks 0 and 1), with their split, and fit
    in shared memory."""
    from test_gpu_tapconv_wstream import check_plan
    sd = O.synthetic_state_dict(17, arch=arch)
    names, code = _engine_names(arch)
    hold = [sd[n].contiguous().float() for n in names]
    ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
    numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
    ctx = C.c_void_p()
    assert emu.vfi_create(0, C.byref(ctx)) == 0, emu.vfi_last_error()
    assert emu.vfi_rife_load(ctx, code, ptrs, numel, len(hold), 0 if operand == "float16" else 1) == 0, emu.vfi_last_error()

    def plan(block, layer):
        st, nc, ns, sm, cm, ws, mc = C.c_int(), C.c_int(), C.c_int(), C.c_int(), C.c_int(), C.c_int(), C.c_int64()
        assert emu.vfi_rife46_layer_plan(ctx, block, layer, C.byref(st), C.byref(nc), C.byref(ns), C.byref(sm),
                                         C.byref(mc), C.byref(cm), C.byref(ws)) == 0, emu.vfi_last_error()
        return dict(stages=st.value, n_cta=nc.value, nsplit=ns.value, smem_bytes=sm.value, cmajor=bool(cm.value),
                    wstream=bool(ws.value))

    try:
        check_plan(plan, arch)
    finally:
        assert emu.vfi_destroy(ctx) == 0


def test_load_refuses_a_wrong_checkpoint(emu):
    sd = O.synthetic_state_dict(0, 1.0)
    names, code = _engine_names("4.6")
    hold = [sd[n].contiguous().float() for n in names]
    ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
    numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
    ctx = C.c_void_p()
    assert emu.vfi_create(0, C.byref(ctx)) == 0
    assert emu.vfi_rife_load(ctx, 47, ptrs, numel, len(hold), 0) != 0      # 4.6 tensors offered as arch 4.7
    assert len(emu.vfi_last_error()) > 0
    out = torch.zeros(1, 64, 64, 3)
    fr = torch.zeros(2, 64, 64, 3)
    f0, f1, ts = np.zeros(1, np.int32), np.ones(1, np.int32), np.asarray([0.5], np.float32)
    vp = lambda x: x.ctypes.data_as(C.c_void_p)   # noqa: E731
    assert emu.vfi_rife46_forward(ctx, C.c_void_p(fr.data_ptr()), 2, 64, 64, 3, vp(f0), vp(f1), vp(ts), 1, C.c_float(1.0),
                                  C.c_void_p(out.data_ptr()), None) != 0   # forward before a successful load
    assert emu.vfi_destroy(ctx) == 0
