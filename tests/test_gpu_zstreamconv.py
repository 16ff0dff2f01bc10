"""-m gpu: streamconv's wgmma kernel (csrc/streamconv.cu, the conv kernel of FILM, Sepconv, FLAVR and IFRNet) per element
against a float64 operator, through the generic hook vfi_streamconv_debug_conv: the case table of
tests/streamconv_util.py (every wgmma N and epilogue, so all 48 kernel instantiations; every padding form, temporal taps,
two sources and channel slices, image sizes down to 1 x 1, grids that make each CTA walk many passes), guard images and
sentinels around every output, two runs bit-identical, the launcher's refusals, and every layer geometry the four
models ship.  The bound and the reference are described in streamconv_util.py; the CUDA-core checker runs the same table
here and on the CPU (test_streamconv_host.py)."""
import pytest
import torch

import streamconv_util as U

pytestmark = pytest.mark.gpu

WORST = {}      # (impl, dtype, ext) -> worst error / bound


@pytest.fixture(scope="module")
def L(pkg):
    from cfi_b200._lib import lib
    yield U.bind(lib())
    for (impl, dtype, ext), r in sorted(WORST.items()):
        print(f"{'wgmma' if impl == 0 else 'checker'} {dtype} ext {ext}: worst error / bound {r:.3f}")


def _run(L, c, dtype, impl, seed, determinism=False, num_sms=None):
    tdt = U.DTYPES[dtype][1]
    r = U.check_case(L, c, tdt, "cuda", impl, seed=seed, num_sms=num_sms, determinism=determinism,
                     stream=torch.cuda.current_stream().cuda_stream)
    key = (impl, dtype, c["ext"])
    WORST[key] = max(WORST.get(key, 0.0), r["ratio16"], r["ratio32"])
    print(f"{c['name']} {dtype} impl {impl}: worst error / bound {r['ratio16']:.3f} (16-bit), {r['ratio32']:.3f} (fp32)")
    return r


@pytest.mark.parametrize("dtype", list(U.DTYPES))
@pytest.mark.parametrize("c", U.CASES, ids=[c["name"] for c in U.CASES])
def test_kernel_meets_the_bound(L, c, dtype):
    """The wgmma kernel, run twice: every element within the bound, guards intact, both runs bit-identical (the kernel
    has no atomics, so a difference is a race)."""
    _run(L, c, dtype, 0, seed=len(c["name"]), determinism=True)


@pytest.mark.parametrize("dtype", list(U.DTYPES))
@pytest.mark.parametrize("c", U.CASES, ids=[c["name"] for c in U.CASES])
def test_checker_meets_the_bound(L, c, dtype):
    _run(L, c, dtype, 1, seed=len(c["name"]))


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("name,change,why", U.REFUSALS, ids=[r[0] for r in U.REFUSALS])
def test_refusals_leave_the_output_untouched(L, name, change, why, impl):
    U.check_refusal(L, U.case(name, **change), torch.float16, "cuda", impl, why)


# ---------------------------------------------------------------------------------------------- shipped geometries
def _film(dtype):
    from cfi_b200._lib import VfiError
    from cfi_b200.engine import FilmEngine
    from oracle import film as OF
    eng = FilmEngine(OF.synthetic_state_dict(0), 0, dtype)
    out = []
    for group, n in ((0, 8), (1, 16), (2, 12)):
        for layer in range(n):
            try:
                p = eng.layer_plan(group, layer)
            except VfiError:
                continue
            c = U.case(f"film_{group}_{layer}", ksize=p["ksize"], c0=p["c0"], c1=p["c1"], n_total=p["n_total"])
            # 1080p (one pair): extract j runs first at level j on both images, flow predictor p < 3 at level p (the
            # shared one from level 3), fusion k at level 3 - k; level l is (1080 >> l) x (1920 >> l)
            lvl, B = ((layer // 2, 2) if group == 0 else (min(layer // 4, 3), 1) if group == 1 else (3 - layer // 3, 1))
            out.append((c, p, dict(B=B, H=1080 >> lvl, W=1920 >> lvl)))
    eng.close()
    return out


def _sepconv(dtype):
    import ctypes as C

    import numpy as np
    from cfi_b200._lib import check, lib
    from cfi_b200.engine import sepconv_state_dict_names
    from oracle import sepconv as OS
    sd = OS.synthetic_state_dict(0)
    op = U.DTYPES[dtype][0]
    h = [1080]
    w = [1920]
    for r in range(1, 5):
        h.append((h[-1] + 1) // 2)
        w.append((w[-1] + 1) // 2)
    out = []
    for name in sepconv_state_dict_names():
        t = sd[name]
        if name.startswith("netInput") or t.dim() != 4:
            continue
        cout, cin = t.shape[:2]
        stride2 = name.startswith("netEncode") and ".netMain.1." in name
        n_total = (cout + 63) // 64 * 64
        buf = np.zeros(16 * cin * n_total, np.uint16)
        c0, n_cta, nsplit = C.c_int(), C.c_int(), C.c_int()
        wt = t.float().contiguous()
        check(lib().vfi_sepconv_debug_pack_host(int(stride2), cin, cout, n_total, op, wt.data_ptr(), buf.ctypes.data,
                                                buf.size, C.byref(c0), C.byref(n_cta), C.byref(nsplit)))
        c = U.case(f"sepconv_{name}", ksize=2 if stride2 else 3, pad_before=1 if stride2 else -1, c0=c0.value,
                   n_total=n_total, ext=1, act=0, slope=0.25, res=None if stride2 else "sep")
        p = dict(n_cta=n_cta.value, nsplit=nsplit.value)
        # 1080p (one pair): encoder row r at h[r]; Decode.netHor row at h[r]; Decode.netVer.{k} (row 4 - k) at twice the
        # size of the row below it; the heads at full size
        if name.startswith("netEncode"):
            r = int(name.split(".")[3])
        elif name.startswith("netDecode.0.netHor"):
            r = 4 - int(name.split(".")[3])
        elif name.startswith("netDecode.0.netVer"):
            r = 4 - int(name.split(".")[3])
        else:
            r = 0
        if name.startswith("netDecode.0.netVer"):
            geo = dict(B=1, H=2 * h[r + 1], W=2 * w[r + 1])
        else:
            geo = dict(B=1, H=h[r], W=w[r])
        out.append((c, p, geo))
    return out


def _flavr(dtype):
    from cfi_b200._lib import VfiError
    from cfi_b200.engine import FlavrEngine
    from oracle import flavr as OFl
    eng = FlavrEngine(OFl.synthetic_state_dict(0), 0, dtype)
    out = []
    for layer in range(61):
        try:
            p = eng.layer_plan(layer)
        except VfiError:
            continue
        c = U.case(f"flavr_{layer}", ksize=p["ksize"], c0=p["c0"], c1=p["c1"], n_total=p["n_total"], ext=p["ext"], act=0,
                   slope=0.0, pad_before=p["pad_y"], pad_before_x=p["pad_x"], kt=p["kt"], pad_t=p["pad_t"], T_in=p["T_in"],
                   T_out=p["T_out"], B=1)
        # 1080p (frames padded to 1088 x 1920, one window): the grid each layer runs on, as a divisor of the padded frame
        # (encoder layer1..4 at /2, /4, /8, /8; decoder 0 and 1's phases at /8, 2 at /4, 3 and 4's phases at /2;
        # feature_fuse at full size)
        f = ([2, 4, 8, 8][layer // 10] if layer < 40 else
             {0: 8, 1: 8, 2: 4, 3: 2, 4: 2}[(layer - 40) // 4] if layer < 60 else 1)
        out.append((c, p, dict(B=1, H=1088 // f, W=1920 // f)))
    eng.close()
    return out


def _ifrnet(variant, dtype):
    from cfi_b200._lib import VfiError
    from cfi_b200.engine import IfrnetEngine, ifrnet_geometry
    from oracle import ifrnet as OI
    eng = IfrnetEngine(OI.synthetic_state_dict(variant, 0), 0, dtype)
    g = ifrnet_geometry(1080, 1920, 1.0)
    grid = {1: (g["h1"], g["w1"]), 2: (g["h2"], g["w2"]), 3: (g["h3"], g["w3"]), 4: (g["h4"], g["w4"])}
    dec = [(g["h4"], g["w4"]), (g["dh3"], g["dw3"]), (g["dh2"], g["dw2"]), (g["dh1"], g["dw1"])]
    out = []
    for layer in range(50):
        try:
            p = eng.layer_plan(layer)
        except VfiError:
            continue
        nf = p["n_f32"]
        c = U.case(f"ifrnet{variant}_{layer}", ksize=p["ksize"], c0=p["c0"], c1=p["c1"], n_total=p["n_total"], ext=2,
                   act=0, n_f32=nf, pad_before=p["pad_y"], pad_before_x=p["pad_x"], res="sep", f32_off=0, f32_pitch=8)
        # 1080p at resize factor 1: encoder pyramid1.1 on level 1, pyramid{l+1}.{0,1} (ids 2l - 1, 2l) on level l + 1;
        # decoder k (ids 10 + 10 k ..) on its grid
        hw = grid[1 if layer == 0 else (layer + 1) // 2 + 1] if layer < 10 else dec[(layer - 10) // 10]
        out.append((c, p, dict(B=1, H=hw[0], W=hw[1])))
    eng.close()
    return out


@pytest.fixture(scope="module")
def shipped(L):
    """model -> [(case, plan of the hook, 1080p geometry)] of every streamconv layer the model ships (fp16 engines: the
    plan does not depend on the operand type).  The hook must plan each one exactly as the model's own layer is planned."""
    raw = {"film": _film("float16"), "sepconv": _sepconv("float16"), "flavr": _flavr("float16"),
           "ifrnet_S": _ifrnet("S", "float16"), "ifrnet_L": _ifrnet("L", "float16")}
    out = {}
    for model, rows in raw.items():
        out[model] = []
        for c, p, geo in rows:
            q = U.plan(L, c)
            assert q is not None, c["name"]
            for key in ("n_cta", "nsplit", "a_slots", "b_slots", "smem_bytes"):
                assert q[key] == p.get(key, q[key]), (c["name"], key, q[key], p[key])
            if "pad_y" in p:
                assert (-q["halo_y0"], -q["halo_x0"]) == (p["pad_y"], p["pad_x"]), c["name"]
            out[model].append((c, q, geo))
    return out


def _k(c):
    return c["kt"] * c["ksize"] ** 2 * (c["c0"] + c["c1"])


def test_every_model_ships_streamconv_layers(shipped):
    counts = {m: len(rows) for m, rows in shipped.items()}
    print("streamconv layers per model:", counts)
    assert all(n > 0 for n in counts.values()), counts


@pytest.mark.parametrize("dtype", list(U.DTYPES))
def test_every_shipped_geometry(L, shipped, dtype):
    """Each distinct layer geometry of the four models, random weights, at a moderate shape (2 tiles x 2 tiles and a
    ragged edge), default grid."""
    seen = {}
    for rows in shipped.values():
        for c, _, _ in rows:
            key = (tuple(U.spec_of(c)), c["res"])
            seen.setdefault(key, c)
    for i, c in enumerate(seen.values()):
        _run(L, dict(c, H=21, W=13), dtype, 0, seed=100 + i)
    print(f"{len(seen)} distinct shipped geometries, {dtype}")


@pytest.mark.parametrize("model", ["film", "sepconv", "flavr", "ifrnet_S", "ifrnet_L"])
def test_largest_layer_at_1080p(L, shipped, model):
    """Each model's largest-K layer at the size it runs at for a 1080p input, default grid, fp16 (bf16 for FILM's:
    its end-to-end check runs fp16 only); the reference is computed on the GPU in float64."""
    c, _, geo = max(shipped[model], key=lambda r: (_k(r[0]), r[2]["H"] * r[2]["W"]))
    dtype = "bfloat16" if model == "film" else "float16"
    r = _run(L, dict(c, **geo, name=c["name"] + "_1080p"), dtype, 0, seed=7)
    print(f"{model}: {c['name']} K = {_k(c)} at {geo}: worst error / bound {r['ratio16']:.3f}")


def test_case_table_covers_every_shipped_plan(L, shipped):
    """Every (n_cta, nsplit, ksize, pad, kt, ext, a_slots, b_slots) a model ships is the plan of some case of the designed
    table (planned, not run): a new layer whose plan the table lacks fails here until a case is added for it."""
    table = {U.plan_key(c, U.plan(L, c)) for c in U.CASES}
    missing = sorted({U.plan_key(c, p) for rows in shipped.values() for c, p, _ in rows} - table)
    assert not missing, f"shipped plans without a case in the table: {missing}"
