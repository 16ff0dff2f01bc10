"""The coarse-span schedule of vfi_rife46_forward on the CPU (csrc/rife46.cu compiled for the host, as in
tests/test_rife_full_host.py): the coarse blocks run over a span of several passes at once, the dense blocks pass by pass.
The first dense block runs over middle spans inside them.
Per-pair arithmetic does not depend on how many pairs a launch covers, so a call with many tasks must give, bit for bit,
the frames of one call per task, and its debug state must be that of a call holding only its last pass's tasks.

The emulator is built with small span budgets, so that frames of 64 x 64 already take several coarse spans; the
profile's span counts show how many each call ran."""
import ctypes as C
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import rife46 as O  # noqa: E402

CUDA_INC = "/usr/local/cuda/include"
BUDGETS = {"small": (256 << 10, 1 << 20), "large": (1 << 20, 4 << 20)}  # (coarse, middle) workspace bytes per span
BATCH = 2
N_FRAMES = 5
N_TASKS = 11  # a multiple of neither the pass width nor any coarse width the budgets give here

# (arch, scale_factor, h, w, budget, operand): coarse blocks 0-1 (4.6 / 4.7 / 4.17 at 1), 0-2 (4.26; scale_factor 0.5),
# 0-3 (4.26 at 0.5), block 0 alone (scale_factor 2 / 4); both operand types on the two block-count families.  Each budget
# is picked so that the case takes two coarse spans.
CASES = [("4.6", 1.0, 64, 64, "small", "float16"), ("4.6", 1.0, 64, 64, "small", "bfloat16"),
         ("4.6", 0.5, 64, 64, "small", "float16"), ("4.6", 2.0, 37, 60, "small", "float16"),
         ("4.6", 4.0, 37, 60, "large", "float16"), ("4.7", 1.0, 50, 64, "small", "float16"),
         ("4.17", 1.0, 64, 50, "small", "float16"), ("4.26", 1.0, 64, 64, "small", "float16"),
         ("4.26", 1.0, 64, 64, "small", "bfloat16"), ("4.26", 0.5, 100, 120, "large", "float16")]


@pytest.fixture(scope="module")
def emus(tmp_path_factory):
    if not (shutil.which("g++") and os.path.exists(os.path.join(CUDA_INC, "cuda_fp16.h"))):
        pytest.skip("g++ / CUDA headers not available")
    d = tmp_path_factory.mktemp("emu_coarse")
    src = os.path.join(ROOT, "tests", "host_emu", "rife_full_emu.cpp")

    def build(item):
        name, (coarse, mid) = item
        so = str(d / f"librife_{name}.so")
        r = subprocess.run(["g++", "-O2", "-std=c++20", "-shared", "-fPIC", "-pthread", "-I" + CUDA_INC,
                            f"-DVFI_COARSE_BUDGET_BYTES={coarse}ull", f"-DVFI_MID_BUDGET_BYTES={mid}ull", "-o", so, src],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
        L = C.CDLL(so)
        L.vfi_last_error.restype = C.c_char_p
        return name, L

    with ThreadPoolExecutor(len(BUDGETS)) as ex:
        return dict(ex.map(build, BUDGETS.items()))


def _vp(x):
    return x.ctypes.data_as(C.c_void_p)


class Ctx:
    def __init__(self, L, arch, sd, operand):
        import __graft_entry__ as ge
        ge.load_package()
        from cfi_b200.engine import ARCH_CODE, state_dict_names
        self.L = L
        hold = [sd[n].contiguous().float() for n in state_dict_names(arch)]
        ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
        numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
        self.ctx = C.c_void_p()
        assert L.vfi_create(0, C.byref(self.ctx)) == 0, L.vfi_last_error()
        assert L.vfi_rife_load(self.ctx, ARCH_CODE[arch], ptrs, numel, len(hold),
                               0 if operand == "float16" else 1) == 0, L.vfi_last_error()
        assert L.vfi_set_batch(self.ctx, BATCH) == 0, L.vfi_last_error()

    def forward(self, fr, f0, f1, ts, sf):
        n, h, w, c = fr.shape
        f0, f1 = np.ascontiguousarray(f0, np.int32), np.ascontiguousarray(f1, np.int32)
        t = np.ascontiguousarray(ts, np.float32)
        out = torch.zeros(len(t), h, w, 3)
        assert self.L.vfi_rife46_forward(self.ctx, C.c_void_p(fr.data_ptr()), n, h, w, c, _vp(f0), _vp(f1), _vp(t), len(t),
                                         C.c_float(sf), C.c_void_p(out.data_ptr()), None) == 0, self.L.vfi_last_error()
        return out

    def debug_state(self, batch):
        hp, wp = C.c_int(), C.c_int()
        assert self.L.vfi_rife46_debug_state(self.ctx, None, None, batch, C.byref(hp), C.byref(wp)) == 0
        flow, mask = torch.zeros(batch, hp.value, wp.value, 4), torch.zeros(batch, hp.value, wp.value)
        assert self.L.vfi_rife46_debug_state(self.ctx, C.c_void_p(flow.data_ptr()), C.c_void_p(mask.data_ptr()), batch,
                                             C.byref(hp), C.byref(wp)) == 0, self.L.vfi_last_error()
        return flow, mask

    def profiled_spans(self, *args):
        """(out, {group id: span count}) of one forward call with the per-group profile on."""
        assert self.L.vfi_rife_profile(self.ctx, 1) == 0
        out = self.forward(*args)
        ids, ms, cnt, n = np.zeros(64, np.int32), np.zeros(64, np.float32), np.zeros(64, np.int32), C.c_int()
        assert self.L.vfi_rife_profile_read(self.ctx, _vp(ids), _vp(ms), _vp(cnt), 64, C.byref(n)) == 0
        assert self.L.vfi_rife_profile(self.ctx, 0) == 0
        return out, {int(ids[i]): int(cnt[i]) for i in range(n.value)}

    def close(self):
        assert self.L.vfi_destroy(self.ctx) == 0


def _tasks(seed):
    """Mixed pairs (not in frame order) and timesteps."""
    rng = np.random.default_rng(seed)
    f0 = rng.integers(0, N_FRAMES - 1, N_TASKS).astype(np.int32)
    f1 = (f0 + 1).astype(np.int32)
    f0[3], f1[3] = f1[3], f0[3]  # one pair backwards
    ts = rng.uniform(0.02, 0.98, N_TASKS).astype(np.float32)
    return f0, f1, ts


def _tiers(arch, sf):
    """(first dense block, the block of the middle spans or None, number of blocks)"""
    s = [(1 << (len(O.SCALE_LIST[arch]) - 1 - i)) / sf for i in range(len(O.SCALE_LIST[arch]))]
    dense = next(i for i in range(1, len(s)) if s[i] <= 2)
    return dense, (dense if dense + 1 < len(s) else None), len(s)


@pytest.mark.parametrize("arch,sf,h,w,budget,operand", CASES, ids=[f"{a}-sf{sf:g}-{h}x{w}-{op}" for a, sf, h, w, _, op in CASES])
def test_coarse_spans_match_one_call_per_task(emus, arch, sf, h, w, budget, operand):
    seed = O.SCALE_LIST[arch][0] * 7 + h + w
    sd = O.synthetic_state_dict(11, 3.0, arch=arch)
    fr = O.synthetic_clip(N_FRAMES, h, w, seed=int(seed)).contiguous()
    f0, f1, ts = _tasks(int(seed))
    e = Ctx(emus[budget], arch, sd, operand)
    try:
        got, spans = e.profiled_spans(fr, f0, f1, ts, sf)
        dense, mid, nb = _tiers(arch, sf)
        n_spans, n_passes = spans[0], spans[90]
        # several coarse spans of several passes each, the first dense block over spans of their own in between, and the
        # passes where they fall when every block runs pass by pass
        assert 2 <= n_spans < n_passes, spans
        assert n_passes == -(-N_TASKS // BATCH), spans
        for i in range(nb):
            if i == mid:
                assert n_spans <= spans[10 * i + 3] <= n_passes, (i, spans)
            else:
                assert spans[10 * i + 3] == (n_spans if i < dense else n_passes), (i, spans)
        last = (N_TASKS - 1) // BATCH * BATCH  # the last pass: tasks [last, N_TASKS)
        flow, mask = e.debug_state(N_TASKS - last)
        for i in range(N_TASKS):
            one = e.forward(fr, f0[i:i + 1], f1[i:i + 1], ts[i:i + 1], sf)
            assert torch.equal(got[i], one[0]), f"task {i} (pair {f0[i]}->{f1[i]}, t={ts[i]:.3f}) differs"
        e.forward(fr, f0[last:], f1[last:], ts[last:], sf)
        flow1, mask1 = e.debug_state(N_TASKS - last)
        assert torch.equal(flow, flow1) and torch.equal(mask, mask1), "debug state is not the last pass's"
    finally:
        e.close()
