"""The FILM path on the CPU against float64 references, in fp16 and bf16 (tests/film16_util.py): every kernel of
csrc/film_elem.cu through vfi_film_debug_elem, per element within its a-priori bound, with guarded outputs; the refusals
of the launchers; and the whole path (csrc/film.cu's schedule, every conv on streamconv's CUDA-core checker) against the
16-bit-faithful oracle, frame and the flows of all 7 levels of both directions (vfi_film_debug_state), per pixel.  All of
it is the library compiled for the host (tests/host_emu/film_full_emu.cpp)."""
import ctypes as C
import os
import shutil
import subprocess

import pytest
import torch

import film16_util as U

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = "/usr/local/cuda/include"
OPERANDS = list(U.DTYPES)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if not (shutil.which("g++") and os.path.exists(os.path.join(CUDA_INC, "cuda_fp16.h"))):
        pytest.skip("g++ / CUDA headers not available")
    so = str(tmp_path_factory.mktemp("emu") / "libfilm16.so")
    src = os.path.join(ROOT, "tests", "host_emu", "film_full_emu.cpp")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-I" + CUDA_INC, "-o", so, src]
                       + os.environ.get("VFI_EMU_CXXFLAGS", "").split(), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(so)
    L.emu_film_open.restype = C.c_void_p
    L.emu_film_open.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    L.emu_film_close.argtypes = [C.c_void_p]
    L.vfi_last_error.restype = C.c_char_p
    L.vfi_film_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                   C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.vfi_film_debug_state.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int),
                                       C.POINTER(C.c_int)]
    return L


class Ctx:
    """A loaded emulated context (every conv on the checker)."""

    def __init__(self, L, sd, operand):
        from cfi_b200.engine import film_state_dict_names
        self.hold = [sd[n].contiguous().float() for n in film_state_dict_names()]
        ptrs = (C.c_void_p * len(self.hold))(*[t.data_ptr() for t in self.hold])
        numel = (C.c_int64 * len(self.hold))(*[t.numel() for t in self.hold])
        self.L = L
        self.ctx = L.emu_film_open(ptrs, numel, len(self.hold), U.DTYPES[operand][0])
        assert self.ctx, L.vfi_last_error()

    def close(self):
        self.L.emu_film_close(self.ctx)


SD = None


def _sd():
    global SD
    if SD is None:
        from oracle import film as OF
        SD = OF.synthetic_state_dict(3, 2.0)
    return SD


@pytest.fixture(scope="module")
def ctxs(emu, pkg):
    cs = {op: Ctx(emu, _sd(), op) for op in OPERANDS}
    yield cs
    for c in cs.values():
        c.close()


@pytest.mark.parametrize("operand", OPERANDS)
@pytest.mark.parametrize("cid,fn,kw", [pytest.param(*c, id=c[0]) for c in U.kernel_cases()])
def test_film_kernel_meets_the_bound_on_host(emu, ctxs, cid, fn, kw, operand):
    E = U.Elem(emu, ctxs[operand].ctx, "cpu")
    r = U.run_kernel_case(E, fn, dict(kw), U.DTYPES[operand][1], "cpu", _sd())
    print(f"{cid} {operand}: worst error / bound {r:.3f}")


@pytest.mark.parametrize("cid,kw,why", [pytest.param(*c, id=c[0]) for c in U.refusal_cases()])
def test_film_kernel_refusals_on_host(emu, ctxs, cid, kw, why):
    U.check_refusal(U.Elem(emu, ctxs["float16"].ctx, "cpu"), "cpu", dict(kw), why)


def run_path(L, sd, fr, operand):
    """One emulated vfi_film_forward of the pair (0, 1), unclamped: (frame [1,h,w,3], flows[dir][level])."""
    c = Ctx(L, sd, operand)
    try:
        fr = fr.contiguous()
        n, h, w, ch = fr.shape
        out = torch.zeros(1, h, w, 3)
        f0, f1 = (C.c_int32 * 1)(0), (C.c_int32 * 1)(1)
        assert L.vfi_film_forward(c.ctx, fr.data_ptr(), n, h, w, ch, C.cast(f0, C.c_void_p), C.cast(f1, C.c_void_p), 1, 0,
                                  out.data_ptr(), None) == 0, L.vfi_last_error()
        flows = []
        for d in range(2):
            lv = []
            for l in range(U.LEVELS):
                hh, ww = C.c_int(), C.c_int()
                assert L.vfi_film_debug_state(c.ctx, d, l, None, 1, C.byref(hh), C.byref(ww)) == 0, L.vfi_last_error()
                assert (hh.value, ww.value) == (h >> l, w >> l)
                v = torch.zeros(1, hh.value, ww.value, 2)
                assert L.vfi_film_debug_state(c.ctx, d, l, v.data_ptr(), 1, C.byref(hh), C.byref(ww)) == 0
                lv.append(v)
            flows.append(lv)
        assert L.vfi_film_debug_state(c.ctx, 0, 7, None, 1, C.byref(hh), C.byref(ww)) != 0
        assert L.vfi_film_debug_state(c.ctx, 0, 0, v.data_ptr(), 2, C.byref(hh), C.byref(ww)) != 0   # one pair ran
        return out, flows
    finally:
        c.close()


@pytest.mark.parametrize("operand", OPERANDS)
@pytest.mark.parametrize("case", [pytest.param(c, id=c[0]) for c in U.PATH_CASES])
def test_film_whole_path_on_host_matches_faithful_oracle(emu, pkg, case, operand):
    sd, fr = U.path_inputs(case)
    got = run_path(emu, sd, fr, operand)
    want = U.path_oracle(sd, fr, [0], [1], operand)
    tf, tv = U.tol(case[0], operand)
    lines, fails, ef, ev = U.path_compare(f"{case[0]} {operand}", got, want, case[1], case[2], tf, tv)
    print("\n".join(lines))
    print(f"OBSERVED {case[0]} {operand}: frame {ef:.2e} flow {ev:.2e}")
    assert not fails, "\n".join(fails)
