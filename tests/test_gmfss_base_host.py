"""The GMFSS Fortuna base model (the `GMFSS_fortuna` checkpoint: no RIFE sub-model, a 12-channel GridNet head) on the CPU:
the product's own `gmfss.GMFSS` schedule over csrc/gmops.cu compiled for the host (tests/host_emu/gmops_emu.cpp), with the
oracle's soft splat (it has its own GPU tests) and no RIFE, against outputs of the UNMODIFIED reference model
(tests/golden/gmfss_base_*.npz).  Also the node's checkpoint table and a whole node call that selects `GMFSS_fortuna`."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden_gmfss import gmfss_cases  # noqa: E402
from oracle import film as OF  # noqa: E402
from oracle import gmfss_base as GB  # noqa: E402
from oracle import gmfss_weights as GW  # noqa: E402
from oracle import ops_ref  # noqa: E402
from oracle import rife46 as R  # noqa: E402

CUDA_INC = "/usr/local/cuda/include"
CASES = gmfss_cases("base")
# vfi_models/gmfss_fortuna/__init__.py:11-25 of the reference, in its order
REF_CKPTS = {
    "GMFSS_fortuna_union": {
        "ifnet": ("rife", "rife46.pth"),
        "flownet": ("gmfss_fortuna", "GMFSS_fortuna_flownet.pkl"),
        "metricnet": ("gmfss_fortuna", "GMFSS_fortuna_union_metric.pkl"),
        "feat_ext": ("gmfss_fortuna", "GMFSS_fortuna_union_feat.pkl"),
        "fusionnet": ("gmfss_fortuna", "GMFSS_fortuna_union_fusionnet.pkl"),
    },
    "GMFSS_fortuna": {
        "flownet": ("gmfss_fortuna", "GMFSS_fortuna_flownet.pkl"),
        "metricnet": ("gmfss_fortuna", "GMFSS_fortuna_metric.pkl"),
        "feat_ext": ("gmfss_fortuna", "GMFSS_fortuna_feat.pkl"),
        "fusionnet": ("gmfss_fortuna", "GMFSS_fortuna_fusionnet.pkl"),
    },
}


@pytest.fixture(scope="module")
def emu_lib(tmp_path_factory):
    if not (shutil.which("g++") and os.path.exists(os.path.join(CUDA_INC, "cuda_fp16.h"))):
        pytest.skip("g++ / CUDA headers not available")
    so = str(tmp_path_factory.mktemp("emu") / "libgmopsemu.so")
    src = os.path.join(ROOT, "tests", "host_emu", "gmops_emu.cpp")
    r = subprocess.run(["g++", "-O2", "-std=c++20", "-shared", "-fPIC", "-pthread", "-I" + CUDA_INC, "-o", so, src] +
                       os.environ.get("VFI_EMU_CXXFLAGS", "").split(), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(so)


def _host_model(lib, sds):
    import __graft_entry__ as ge
    ge.load_package()
    from cfi_b200.gmfss import GMFSS, Ops
    return GMFSS(sds, Ops(lib, torch.device("cpu")), splat=lambda x, fl, z: ops_ref.softsplat(x, fl, z, "soft"), rife=None)


def _case(name):
    cfg = CASES[name]
    g = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    sds = GB.synthetic_state_dicts(cfg["seed"])
    fr = OF.synthetic_clip(2, cfg["h"], cfg["w"], seed=cfg["clip_seed"]).permute(0, 3, 1, 2).contiguous()
    return cfg, g, sds, fr


@pytest.mark.parametrize("name", sorted(CASES)[:1])
def test_base_model_on_the_product_kernels(emu_lib, name):
    """GMFSS.reuse (flows, metrics) and GMFSS.inference (12-channel GridNet input) on the padded 70x100 pair, against the
    unmodified reference; the node test below runs the 96x128 case through GMFSS.interpolate's padding and crop"""
    cfg, g, sds, fr = _case(name)
    m = _host_model(emu_lib, sds)
    assert m.variant == "base" and m.rife is None
    h, w = cfg["h"], cfg["w"]
    ph, pw = ((h - 1) // 64 + 1) * 64, ((w - 1) // 64 + 1) * 64
    i0, i1 = F.pad(fr[0:1], (0, pw - w, 0, ph - h)).contiguous(), F.pad(fr[1:2], (0, pw - w, 0, ph - h)).contiguous()
    state = m.reuse(i0, i1)
    ef = max((state[k] - torch.from_numpy(g[n])).abs().max().item() for k, n in ((0, "flow01"), (1, "flow10")))
    em = max((state[k] - torch.from_numpy(g[n])).abs().max().item() for k, n in ((2, "metric0"), (3, "metric1")))
    out = m.inference(state, cfg["t"])[:, :, :h, :w]
    ref = torch.from_numpy(g["out"])
    assert out.shape == ref.shape
    p = R.psnr(out, ref)
    print(f"{name}: base GMFSS on the product kernels (host build): flows within {ef:.2e} px, metrics within {em:.2e}, "
          f"frame PSNR {p:.1f} dB")
    assert ef <= 2e-2 and em <= 1e-2 and p >= 50.0   # the GPU test's flow bound; fp32 reordering in the global softmax


def test_variant_follows_the_weights(emu_lib):
    """no ifnet -> base; a GridNet that does not match the variant the weights imply is refused at construction"""
    base = GB.synthetic_state_dicts(0)
    union = GW.synthetic_state_dicts(0)
    assert _host_model(emu_lib, base)._head == "head"
    assert _host_model(emu_lib, union).variant == "union"
    with pytest.raises(KeyError, match="residual_model_head"):
        _host_model(emu_lib, {**base, "ifnet": union["ifnet"]})            # a base GridNet under the union schedule
    with pytest.raises(KeyError, match="residual_model_head"):
        _host_model(emu_lib, {k: v for k, v in union.items() if k != "ifnet"})


def test_node_checkpoint_table_is_the_references():
    import __graft_entry__ as ge
    ge.load_package()
    import cfi_b200 as P
    import cfi_b200.gmfss_node as GN
    assert list(GN.CKPTS_PATH_CONFIG) == ["GMFSS_fortuna_union", "GMFSS_fortuna"]
    assert GN.CKPTS_PATH_CONFIG == REF_CKPTS
    assert list(GN.CKPTS_PATH_CONFIG["GMFSS_fortuna"]) == ["flownet", "metricnet", "feat_ext", "fusionnet"]
    assert GN.GMFSS_Fortuna_VFI.INPUT_TYPES()["required"]["ckpt_name"] == (["GMFSS_fortuna_union", "GMFSS_fortuna"],)
    assert P.NODE_CLASS_MAPPINGS["GMFSS Fortuna VFI"] is GN.GMFSS_Fortuna_VFI


def test_node_selects_the_base_checkpoint(emu_lib, tmp_path, monkeypatch):
    """a graph that picks `GMFSS_fortuna`: the node loads the four checkpoint files (DataParallel 'module.' prefixes
    stripped), builds the base model and returns [(N-1)*m+1, H, W, 3] float32 on the CPU; the middle frame at t = 0.5 is the
    reference's"""
    import __graft_entry__ as ge
    ge.load_package()
    import cfi_b200.gmfss as G
    import cfi_b200.gmfss_node as GN
    name = "gmfss_base_96x128_t0.5"
    cfg, g, sds, _ = _case(name)
    asked = []
    for key, (kind, fname) in GN.CKPTS_PATH_CONFIG["GMFSS_fortuna"].items():
        os.makedirs(tmp_path / kind, exist_ok=True)
        torch.save({"module." + k: v for k, v in sds[key].items()}, str(tmp_path / kind / fname))

    def fetch(kind, fname):
        asked.append(fname)
        return str(tmp_path / kind / fname)

    built = []

    def build(sds_, device=0):
        built.append(sorted(sds_))
        return _host_model(emu_lib, sds_)

    monkeypatch.setattr(GN, "load_file_from_github_release", fetch)
    monkeypatch.setattr(G, "build_gpu_model", build)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(GN, "_model_cache", {})
    fr = OF.synthetic_clip(2, cfg["h"], cfg["w"], seed=cfg["clip_seed"])
    (out,) = GN.GMFSS_Fortuna_VFI().vfi("GMFSS_fortuna", fr, multiplier=2)
    assert sorted(asked) == sorted(f for _, f in REF_CKPTS["GMFSS_fortuna"].values())
    assert built == [["feat_ext", "flownet", "fusionnet", "metricnet"]]
    assert out.shape == (3, cfg["h"], cfg["w"], 3) and out.dtype == torch.float32 and not out.is_cuda
    assert torch.equal(out[0], fr[0]) and torch.equal(out[2], fr[1])
    p = R.psnr(out[1].permute(2, 0, 1)[None], torch.from_numpy(g["out"]))
    print(f"GMFSS_fortuna node on the host build: PSNR {p:.1f} dB")
    assert p >= 50.0
    assert GN._load_model("GMFSS_fortuna") is GN._model_cache["GMFSS_fortuna"] and len(built) == 1   # cached by name
