"""The tap-conv plan of every IFBlock layer the library builds at load time (csrc/rife46.cu: the plan table and the layer
constructor), read back through vfi_rife46_layer_plan from the host emulation, against a stored table
(tests/golden/rife_layer_plans.json): stages, n_cta, nsplit, smem_bytes, macs_per_cell, cmajor and wstream of each
(block, layer) of RIFE 4.6, 4.7, 4.17 and 4.26 with fp16 and bf16 operands.  A plan change shows here as a diff of this
table, on the CPU."""
import ctypes as C
import json
import os

import pytest

from oracle import rife46 as O
from test_rife_full_host import ROOT, _engine_names, emu  # noqa: F401  (emu: the module-scoped host-emulation fixture)

with open(os.path.join(ROOT, "tests", "golden", "rife_layer_plans.json")) as fh:
    PLANS = json.load(fh)


@pytest.mark.parametrize("operand", ["float16", "bfloat16"])
@pytest.mark.parametrize("arch", ["4.6", "4.7", "4.17", "4.26"])
def test_block_layer_plans_match_stored_table(emu, arch, operand):  # noqa: F811
    sd = O.synthetic_state_dict(17, arch=arch)
    names, code = _engine_names(arch)
    hold = [sd[n].contiguous().float() for n in names]
    ptrs = (C.c_void_p * len(hold))(*[t.data_ptr() for t in hold])
    numel = (C.c_int64 * len(hold))(*[t.numel() for t in hold])
    ctx = C.c_void_p()
    assert emu.vfi_create(0, C.byref(ctx)) == 0, emu.vfi_last_error()
    try:
        assert emu.vfi_rife_load(ctx, code, ptrs, numel, len(hold), 0 if operand == "float16" else 1) == 0, \
            emu.vfi_last_error()
        want = PLANS[arch][operand]
        for b, layers in enumerate(want):
            for l, row in enumerate(layers):
                v = [C.c_int() for _ in range(4)] + [C.c_int64()] + [C.c_int() for _ in range(2)]
                assert emu.vfi_rife46_layer_plan(ctx, b, l, *[C.byref(x) for x in v]) == 0, emu.vfi_last_error()
                got = [x.value for x in v]
                assert got == row, (arch, operand, b, l, dict(zip(PLANS["fields"], got)), dict(zip(PLANS["fields"], row)))
            # the table lists every layer of the block: the next index is refused
            assert emu.vfi_rife46_layer_plan(ctx, b, len(layers), None, None, None, None, None, None, None) != 0
        assert emu.vfi_rife46_layer_plan(ctx, len(want), 0, None, None, None, None, None, None, None) != 0
    finally:
        assert emu.vfi_destroy(ctx) == 0
