"""The Sepconv path on the CPU against float64 references, in fp16 and bf16 (tests/sepconv16_util.py): every kernel of
csrc/sepconv_elem.cu through vfi_sepconv_debug_elem, per element within its a-priori bound, with guarded outputs, and the
hook's refusals; the separable-convolution op of csrc/ops.cu (PY = 2 in this process, PY = 1 and 3 in one subprocess
each); and the whole path (csrc/sepconv.cu's schedule, every conv on streamconv's CUDA-core checker) split at the
coefficients: planes and rows (vfi_sepconv_debug_state) against the 16-bit-faithful oracle, the frame against float64
arithmetic on the library's coefficients and against the oracle.  All of it is the library compiled for the host
(tests/host_emu/sepconv_full_emu.cpp).  A few minutes of CPU time, most of it in the whole-path cases."""
import ctypes as C
import os
import shutil
import subprocess

import pytest
import torch

import sepconv16_util as U

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = "/usr/local/cuda/include"
OPERANDS = list(U.DTYPES)


@pytest.fixture(scope="module")
def emu_so(tmp_path_factory):
    if not (shutil.which("g++") and os.path.exists(os.path.join(CUDA_INC, "cuda_fp16.h"))):
        pytest.skip("g++ / CUDA headers not available")
    so = str(tmp_path_factory.mktemp("emu") / "libsepconv16.so")
    src = os.path.join(ROOT, "tests", "host_emu", "sepconv_full_emu.cpp")
    r = subprocess.run(["g++", "-O2", "-std=c++20", "-shared", "-fPIC", "-pthread", "-I" + CUDA_INC, "-o", so, src]
                       + os.environ.get("VFI_EMU_CXXFLAGS", "").split(), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return so


@pytest.fixture(scope="module")
def emu(emu_so):
    L = C.CDLL(emu_so)
    L.emu_sepconv_open.restype = C.c_void_p
    L.emu_sepconv_open.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    L.emu_sepconv_close.argtypes = [C.c_void_p]
    L.emu_sepconv_op.argtypes = [C.c_void_p] * 4 + [C.c_int] * 6
    L.vfi_last_error.restype = C.c_char_p
    L.vfi_sepconv_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                      C.c_int, C.c_void_p, C.c_void_p]
    L.vfi_sepconv_debug_state.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int)]
    return L


class Ctx:
    """A loaded emulated context (every conv on the checker)."""

    def __init__(self, L, sd, operand):
        from cfi_b200.engine import sepconv_state_dict_names
        self.hold = [sd[n].contiguous().float() for n in sepconv_state_dict_names()]
        ptrs = (C.c_void_p * len(self.hold))(*[t.data_ptr() for t in self.hold])
        numel = (C.c_int64 * len(self.hold))(*[t.numel() for t in self.hold])
        self.L = L
        self.ctx = L.emu_sepconv_open(ptrs, numel, len(self.hold), U.DTYPES[operand][0])
        assert self.ctx, L.vfi_last_error()

    def close(self):
        self.L.emu_sepconv_close(self.ctx)


SD = None


def _sd():
    global SD
    if SD is None:
        from oracle import sepconv as OS
        SD = OS.synthetic_state_dict(3, U.TRUNK_GAIN)
    return SD


@pytest.fixture(scope="module")
def ctxs(emu, pkg):
    cs = {op: Ctx(emu, _sd(), op) for op in OPERANDS}
    yield cs
    for c in cs.values():
        c.close()


@pytest.mark.parametrize("operand", OPERANDS)
@pytest.mark.parametrize("cid,fn,kw", [pytest.param(*c, id=c[0]) for c in U.kernel_cases()])
def test_sepconv_kernel_meets_the_bound_on_host(emu, ctxs, cid, fn, kw, operand):
    E = U.Elem(emu, ctxs[operand].ctx, "cpu")
    r = U.run_kernel_case(E, fn, dict(kw), U.DTYPES[operand][1], "cpu", _sd())
    print(f"{cid} {operand}: worst error / bound {r:.3f}")


@pytest.mark.parametrize("cid,kw,why", [pytest.param(*c, id=c[0]) for c in U.refusal_cases()])
def test_sepconv_kernel_refusals_on_host(emu, ctxs, cid, kw, why):
    U.check_refusal(U.Elem(emu, ctxs["float16"].ctx, "cpu"), "cpu", kw, why)


@pytest.mark.parametrize("case", [pytest.param(c, id=c[0]) for c in U.OP_CASES])
def test_sepconv_op_meets_the_bound_on_host(emu, case):
    run = lambda x, v, h, o, *a: emu.emu_sepconv_op(x.data_ptr(), v.data_ptr(), h.data_ptr(), o, *a)   # noqa: E731
    print(f"op {case[0]}: worst error / bound {U.check_op(run, case, 'cpu'):.3f}")


@pytest.mark.parametrize("py", [1, 3])
def test_sepconv_op_other_row_blockings_on_host(emu_so, py):
    res = U.op_subprocess(py, "host", emu_so)
    print(f"PY {py}: " + ", ".join(f"{k} {v:.3f}" for k, v in res.items()))
    assert max(res.values()) <= 1.0


def run_path(L, sd, fr, operand):
    """One emulated vfi_sepconv_forward of the pair (0, 1): {"frame", "coef", "rows", "stats"}, and the hook's refusals
    after it."""
    c = Ctx(L, sd, operand)
    shape = (C.c_int * 4)()
    try:
        assert L.vfi_sepconv_debug_state(c.ctx, 0, 0, None, 1, shape) != 0     # before any forward
        assert "no forward has run" in L.vfi_last_error().decode()
        fr = fr.contiguous()
        n, h, w, ch = fr.shape
        out = torch.zeros(1, h, w, 3)
        f0, f1 = (C.c_int32 * 1)(0), (C.c_int32 * 1)(1)
        assert L.vfi_sepconv_forward(c.ctx, fr.data_ptr(), n, h, w, ch, C.cast(f0, C.c_void_p), C.cast(f1, C.c_void_p), 1,
                                     out.data_ptr(), None) == 0, L.vfi_last_error()
        tdt = U.DTYPES[operand][1]

        def state(what, index, dt):
            assert L.vfi_sepconv_debug_state(c.ctx, what, index, None, 1, shape) == 0, L.vfi_last_error()
            t = torch.empty(tuple(shape) if what != 2 else (1, 2), dtype=dt)
            assert L.vfi_sepconv_debug_state(c.ctx, what, index, t.data_ptr(), 1, shape) == 0, L.vfi_last_error()
            return t
        got = dict(frame=out, coef=[state(0, k, torch.float32) for k in range(4)],
                   rows=[state(1, r, tdt) for r in U.ROWS], stats=state(2, 0, torch.float64))
        for what, index in ((0, 4), (0, -1), (1, 0), (1, 5), (2, 1), (3, 0)):
            assert L.vfi_sepconv_debug_state(c.ctx, what, index, None, 1, shape) != 0, (what, index)
        assert L.vfi_sepconv_debug_state(c.ctx, 1, 1, out.data_ptr(), 2, shape) != 0     # one pair ran
        assert "batch larger than the last forward" in L.vfi_last_error().decode()
        return got
    finally:
        c.close()


@pytest.mark.parametrize("operand", OPERANDS)
@pytest.mark.parametrize("case", [pytest.param(c, id=c[0]) for c in U.PATH_CASES])
def test_sepconv_whole_path_on_host_matches_faithful_oracle(emu, pkg, case, operand):
    sd, fr = U.path_inputs(case)
    got = run_path(emu, sd, fr, operand)
    want = U.path_oracle(sd, fr, [0], [1], operand)
    label = f"{case[0]} {operand}"
    U.check_stats(got["stats"], want["stats"], label)
    rt = U.check_tail(label, fr, [0], [1], got)
    lines, fails, obs = U.path_compare(label, got, want, case[1], case[2], U.tol(case[0], operand))
    print("\n".join(lines))
    print(f"OBSERVED {case[0]} {operand}: " + ", ".join(f"{v:.2e}" for v in obs) + f"; tail error / bound {rt:.3f}")
    assert not fails, "\n".join(fails)
