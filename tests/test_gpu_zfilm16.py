"""-m gpu: the FILM path on the H100 against float64 references, in fp16 and bf16 (tests/film16_util.py).

In this process: every kernel of csrc/film_elem.cu through vfi_film_debug_elem, per element within its a-priori bound
with guarded outputs, and the launchers' refusals; the whole path (wgmma convs) against the 16-bit-faithful oracle, frame
and the flows of all 7 levels of both directions (vfi_film_debug_state), per pixel, each case within MARGIN (4) x what the
host emulation showed on it; 1080 x 1920 (odd levels 135, 67, 33) within MARGIN x the largest calibrated error, the
oracle in float64 on the GPU after the engine is closed; 16 pairs over 17 frames in one call, each bit-identical to its
own single-pair call; and 17 pairs refused.
"""
import ctypes as C
import time

import pytest
import torch

import film16_util as U

pytestmark = pytest.mark.gpu
OPERANDS = list(U.DTYPES)


@pytest.fixture(scope="module")
def engines(pkg):
    from cfi_b200.engine import FilmEngine
    from oracle import film as OF
    sd = OF.synthetic_state_dict(3, 2.0)
    e = {op: FilmEngine(sd, 0, op) for op in OPERANDS}
    yield sd, e
    for x in e.values():
        x.close()


def _elem(eng):
    from cfi_b200._lib import lib
    return U.Elem(lib(), eng._ctx, "cuda", torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("operand", OPERANDS)
@pytest.mark.parametrize("cid,fn,kw", [pytest.param(*c, id=c[0]) for c in U.kernel_cases()])
def test_film_kernel_meets_the_bound(engines, cid, fn, kw, operand):
    sd, e = engines
    r = U.run_kernel_case(_elem(e[operand]), fn, dict(kw), U.DTYPES[operand][1], "cuda", sd)
    print(f"{cid} {operand}: worst error / bound {r:.3f}")


@pytest.mark.parametrize("cid,kw,why", [pytest.param(*c, id=c[0]) for c in U.refusal_cases()])
def test_film_kernel_refusals(engines, cid, kw, why):
    U.check_refusal(_elem(engines[1]["float16"]), "cuda", dict(kw), why)


def _run(eng, fr, f0, f1):
    """(frames [B,h,w,3] unclamped, flows[dir][level] [B,H_l,W_l,2]) of one forward call."""
    out = eng.forward(fr, f0, f1, clamp=False)
    flows = [[eng.debug_state(d, l, len(f0)) for l in range(U.LEVELS)] for d in range(2)]
    torch.cuda.synchronize()
    return out, flows


def _check(label, got, want, h, w, tf, tv):
    lines, fails, ef, ev = U.path_compare(label, got, want, h, w, tf, tv)
    print("\n".join(lines))
    print(f"{label}: max |err| frame {ef:.3e}, flow {ev:.3e} px (bounds {tf:.3e}, {tv:.3e})")
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("operand", OPERANDS)
@pytest.mark.parametrize("case", [pytest.param(c, id=c[0]) for c in U.PATH_CASES])
def test_film_whole_path_matches_faithful_oracle(pkg, case, operand):
    from cfi_b200.engine import FilmEngine
    sd, fr = U.path_inputs(case)
    eng = FilmEngine(sd, 0, operand)
    try:
        got = _run(eng, fr.cuda().contiguous(), [0], [1])
    finally:
        eng.close()
    want = U.path_oracle(sd, fr, [0], [1], operand, device="cuda")
    _check(f"{case[0]} {operand}", got, want, case[1], case[2], *U.tol(case[0], operand))


@pytest.mark.parametrize("operand", OPERANDS)
def test_film_1080p_matches_faithful_oracle(pkg, operand):
    """No host calibration exists at this size: the bound is MARGIN x the largest error of any calibrated case."""
    from cfi_b200.engine import FilmEngine
    from oracle import film as OF
    sd = OF.synthetic_state_dict(13, 4.0)
    fr = OF.synthetic_clip(2, 1080, 1920, seed=1080)
    t0 = time.time()
    eng = FilmEngine(sd, 0, operand)
    try:
        got = _run(eng, fr.cuda().contiguous(), [0], [1])
    finally:
        eng.close()
    torch.cuda.empty_cache()
    t1 = time.time()
    want = U.path_oracle(sd, fr, [0], [1], operand, device="cuda")
    torch.cuda.synchronize()
    print(f"1080p {operand}: library {t1 - t0:.1f} s, float64 oracle {time.time() - t1:.1f} s")
    assert [v.shape[1:3] for v in got[1][0]] == [(1080 >> l, 1920 >> l) for l in range(U.LEVELS)]
    _check(f"1080x1920 {operand}", got, want, 1080, 1920, *U.tol("1080x1920", operand))


@pytest.mark.parametrize("operand", OPERANDS)
def test_film_16_pairs_in_one_call_equal_single_pairs(pkg, operand):
    """Pairs (i, i + 1) of 17 frames in ONE call (images indexed k * 16 + pair through every buffer) equal the
    single-pair calls bit for bit, frames and flows; 4-channel frames."""
    from cfi_b200.engine import FilmEngine
    from oracle import film as OF
    sd = OF.synthetic_state_dict(14, 2.0)
    fr = torch.cat([OF.synthetic_clip(17, 72, 104, seed=16), torch.ones(17, 72, 104, 1)], -1).cuda().contiguous()
    eng = FilmEngine(sd, 0, operand)
    try:
        f0, f1 = list(range(16)), list(range(1, 17))
        out, flows = _run(eng, fr, f0, f1)
        out, flows = out.clone(), [[v.clone() for v in lv] for lv in flows]
        for i in range(16):
            one, fl1 = _run(eng, fr, [i], [i + 1])
            assert torch.equal(out[i], one[0]), i
            for d in range(2):
                for l in range(U.LEVELS):
                    assert torch.equal(flows[d][l][i], fl1[d][l][0]), (i, d, l)
        # 17 pairs are refused by the library itself (the engine asserts before calling it)
        from cfi_b200._lib import lib
        L = lib()
        big = torch.empty(17, 72, 104, 3, device="cuda")
        a = (C.c_int32 * 17)(*range(16), 0)
        b = (C.c_int32 * 17)(*range(1, 17), 1)
        rc = L.vfi_film_forward(eng._ctx, fr.data_ptr(), 17, 72, 104, 4, C.cast(a, C.c_void_p), C.cast(b, C.c_void_p), 17,
                                0, big.data_ptr(), torch.cuda.current_stream().cuda_stream)
        assert rc != 0 and "n_pairs must be in [1,16]" in L.vfi_last_error().decode()
    finally:
        eng.close()
