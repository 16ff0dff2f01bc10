"""-m gpu: the Sepconv path on the H100 against float64 references, in fp16 and bf16 (tests/sepconv16_util.py).

In this process: every kernel of csrc/sepconv_elem.cu through vfi_sepconv_debug_elem, per element within its a-priori
bound with guarded outputs, and the hook's refusals; the separable-convolution op (vfi_sepconv) at PY = 2, and at PY = 1
and 3 in one subprocess each; the whole path (wgmma convs) split at the coefficients - planes and rows against the
16-bit-faithful oracle within MARGIN (4) x what the host emulation showed on each case, the frame against float64
arithmetic on the library's coefficients within its a-priori bound and against the oracle; 1080 x 1920 (where the
decoder's crop-after-conv path runs at row 3) and 2160 x 3840 (the benchmark's size), the trunk within MARGIN x the
largest calibrated error, the oracle in float64 on the GPU after the engine is closed; 16 pairs over 17 frames in one
call, each bit-identical to its own single-pair call, and 17 pairs refused; the same call twice, bit-identical.
"""
import ctypes as C
import time

import pytest
import torch

import sepconv16_util as U

pytestmark = pytest.mark.gpu
OPERANDS = list(U.DTYPES)


@pytest.fixture(scope="module")
def engines(pkg):
    from cfi_b200.engine import SepconvEngine
    from oracle import sepconv as OS
    sd = OS.synthetic_state_dict(3, U.TRUNK_GAIN)
    e = {op: SepconvEngine(sd, 0, op) for op in OPERANDS}
    yield sd, e
    for x in e.values():
        x.close()


def _elem(eng):
    from cfi_b200._lib import lib
    return U.Elem(lib(), eng._ctx, "cuda", torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("operand", OPERANDS)
@pytest.mark.parametrize("cid,fn,kw", [pytest.param(*c, id=c[0]) for c in U.kernel_cases()])
def test_sepconv_kernel_meets_the_bound(engines, cid, fn, kw, operand):
    sd, e = engines
    r = U.run_kernel_case(_elem(e[operand]), fn, dict(kw), U.DTYPES[operand][1], "cuda", sd)
    print(f"{cid} {operand}: worst error / bound {r:.3f}")


@pytest.mark.parametrize("cid,kw,why", [pytest.param(*c, id=c[0]) for c in U.refusal_cases()])
def test_sepconv_kernel_refusals(engines, cid, kw, why):
    U.check_refusal(_elem(engines[1]["float16"]), "cuda", kw, why)


@pytest.mark.parametrize("case", [pytest.param(c, id=c[0]) for c in U.OP_CASES])
def test_sepconv_op_meets_the_bound(pkg, case):
    print(f"op PY 2 {case[0]}: worst error / bound {U.check_op(U.gpu_op_runner(), case, 'cuda'):.3f}")


@pytest.mark.parametrize("py", [1, 3])
def test_sepconv_op_other_row_blockings(pkg, py):
    res = U.op_subprocess(py, "gpu")
    print(f"op PY {py}: " + ", ".join(f"{k} {v:.3f}" for k, v in res.items()))
    assert max(res.values()) <= 1.0


def _run(eng, fr, f0, f1):
    """{"frame", "coef", "rows", "stats"} of one forward call."""
    out = eng.forward(fr, f0, f1)
    B = len(f0)
    got = dict(frame=out, coef=[eng.debug_state(0, k, B) for k in range(4)], rows=[eng.debug_state(1, r, B) for r in U.ROWS],
               stats=eng.debug_state(2, 0, B))
    torch.cuda.synchronize()
    return got


def _check(label, fr, got, want, h, w, t):
    U.check_stats(got["stats"], want["stats"], label)
    rt = U.check_tail(label, fr, [0], [1], got)
    lines, fails, obs = U.path_compare(label, got, want, h, w, t)
    print("\n".join(lines))
    print(f"{label}: max |err| coef {obs[0]:.3e}, rows " + ", ".join(f"{v:.3e}" for v in obs[1:5]) +
          f", frame {obs[5]:.3e}; worst ratio to the bound trunk {max(o / b for o, b in zip(obs[:5], t[:5])):.2f}, "
          f"frame {obs[5] / t[5]:.2f}, tail {rt:.3f}")
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("operand", OPERANDS)
@pytest.mark.parametrize("case", [pytest.param(c, id=c[0]) for c in U.PATH_CASES])
def test_sepconv_whole_path_matches_faithful_oracle(pkg, case, operand):
    from cfi_b200.engine import SepconvEngine
    sd, fr = U.path_inputs(case)
    eng = SepconvEngine(sd, 0, operand)
    try:
        got = _run(eng, fr.cuda().contiguous(), [0], [1])
    finally:
        eng.close()
    want = U.path_oracle(sd, fr, [0], [1], operand, device="cuda")
    _check(f"{case[0]} {operand}", fr, got, want, case[1], case[2], U.tol(case[0], operand))


@pytest.mark.parametrize("operand", OPERANDS)
@pytest.mark.parametrize("hw", [(1080, 1920), (2160, 3840)], ids=["1080p", "4K"])
def test_sepconv_large_frames_match_faithful_oracle(pkg, hw, operand):
    """No host calibration exists at these sizes: the trunk and the oracle frame are held to MARGIN x the largest error of
    any calibrated case, the tail to its a-priori bound."""
    from cfi_b200.engine import SepconvEngine
    from oracle import sepconv as OS
    h, w = hw
    sd = OS.synthetic_state_dict(31, U.TRUNK_GAIN)
    case = (f"{h}x{w}", h, w, None, U.TRUNK_GAIN, "clip", 3)
    _, fr = U.path_inputs(("clip", h, w, 0, 1.0, "clip", 3))
    torch.cuda.synchronize()
    t0 = time.time()
    eng = SepconvEngine(sd, 0, operand)
    try:
        got = _run(eng, fr.cuda().contiguous(), [0], [1])
        t1 = time.time()
    finally:
        eng.close()
    torch.cuda.empty_cache()
    t2 = time.time()
    want = U.path_oracle(sd, fr, [0], [1], operand, device="cuda")
    torch.cuda.synchronize()
    print(f"{h}x{w} {operand}: library (load + forward + copies) {t1 - t0:.1f} s, float64 oracle {time.time() - t2:.1f} s")
    _check(f"{h}x{w} {operand}", fr, got, want, h, w, U.tol(case[0], operand))


@pytest.mark.parametrize("operand", OPERANDS)
def test_sepconv_16_pairs_in_one_call_equal_single_pairs(pkg, operand):
    """Pairs (i, i + 1) of 17 frames in ONE call equal the single-pair calls bit for bit: frame, coefficient planes and
    rows; 4-channel frames; 17 pairs are refused by the library itself."""
    from cfi_b200.engine import SepconvEngine
    from oracle import sepconv as OS
    sd = OS.synthetic_state_dict(14, U.TRUNK_GAIN)
    g = torch.Generator().manual_seed(17)
    fr = torch.rand(17, 45, 54, 4, generator=g).cuda().contiguous()
    eng = SepconvEngine(sd, 0, operand)
    try:
        f0, f1 = list(range(16)), list(range(1, 17))
        allp = _run(eng, fr, f0, f1)
        allp = {k: ([t.clone() for t in v] if isinstance(v, list) else v.clone()) for k, v in allp.items()}
        for i in range(16):
            one = _run(eng, fr, [i], [i + 1])
            assert torch.equal(allp["frame"][i], one["frame"][0]), i
            for k in range(4):
                assert torch.equal(allp["coef"][k][i], one["coef"][k][0]), (i, k)
            for j in range(4):
                assert torch.equal(allp["rows"][j][i], one["rows"][j][0]), (i, j)
        from cfi_b200._lib import lib
        L = lib()
        big = torch.empty(17, 45, 54, 3, device="cuda")
        a = (C.c_int32 * 17)(*range(16), 0)
        b = (C.c_int32 * 17)(*range(1, 17), 1)
        rc = L.vfi_sepconv_forward(eng._ctx, fr.data_ptr(), 17, 45, 54, 4, C.cast(a, C.c_void_p), C.cast(b, C.c_void_p), 17,
                                   big.data_ptr(), torch.cuda.current_stream().cuda_stream)
        assert rc != 0 and "n_pairs must be in [1,16]" in L.vfi_last_error().decode()
    finally:
        eng.close()


@pytest.mark.parametrize("operand", OPERANDS)
def test_sepconv_same_call_twice_is_bit_identical(pkg, operand):
    """Frame, planes, rows and the per-pair double sums of two identical calls (1080p, 3 pairs) are equal bit for bit."""
    from cfi_b200.engine import SepconvEngine
    from oracle import sepconv as OS
    sd = OS.synthetic_state_dict(15, U.TRUNK_GAIN)
    g = torch.Generator().manual_seed(18)
    fr = torch.rand(4, 1080, 1920, 3, generator=g).cuda().contiguous()
    eng = SepconvEngine(sd, 0, operand)
    try:
        runs = []
        for _ in range(2):
            r = _run(eng, fr, [0, 1, 2], [1, 2, 3])
            runs.append({k: ([t.clone() for t in v] if isinstance(v, list) else v.clone()) for k, v in r.items()})
        a, b = runs
        assert torch.equal(a["stats"], b["stats"]), (a["stats"] - b["stats"]).abs().max()
        assert torch.equal(a["frame"], b["frame"])
        assert all(torch.equal(x, y) for x, y in zip(a["coef"], b["coef"]))
        assert all(torch.equal(x, y) for x, y in zip(a["rows"], b["rows"]))
    finally:
        eng.close()
