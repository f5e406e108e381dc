"""Host-side checks of the tensor-core kernels that need no GPU:

* every kernel that opts in to a large dynamic shared-memory budget stays inside the 227 KB per-block limit TOGETHER with its
  static shared memory (read from the built library with cuobjdump): a kernel over the limit fails every launch with
  `cudaFuncSetAttribute: invalid argument`;
* the host-only plan of the packed-operand family (`mnb_pk_conv_plan`, `mnb_pk_wgrad_scratch_bytes`, `mnb_pk_wimage_bytes`,
  `mnb_pk_act_bytes`) covers every convolution of the BASELINE.json models at their bench shapes, inside shared memory and the
  register budget of the accumulators."""
import ctypes as C
import re
import shutil
import subprocess

import pytest

from tests.pk_plan_util import LIMIT, RESERVED, budget, model_convs

# kernel (mangled-name fragment) -> (source file, name of its dynamic shared-memory budget constant)
BUDGETS = {
    "pk14pk_conv_kernel": ("mnb_pk.cu", "kSmemBudget"),
    "pk15pk_wgrad_kernel": ("mnb_pk.cu", "kSmemBudget"),
    "tcconv14conv_tc_kernel": ("mnb_conv_tc_fwd.cu", "kMaxDynSmem"),
    "tcwgrad15wgrad_tc_kernel": ("mnb_conv_tc_wgrad.cu", "kMaxDynSmem"),
    "tcfp3210fwd_kernel": ("mnb_conv_fp32_tc.cu", "kMaxDynSmem"),
    "tcfp3212wgrad_kernel": ("mnb_conv_fp32_tc.cu", "kMaxDynSmem"),
}


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_static_plus_dynamic_shared_memory_fits_the_block_limit():
    from micronet_b200 import _lib as L
    out = subprocess.run(["cuobjdump", "-res-usage", L.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs = re.findall(r"Function (\S+?):\s*\n\s*(.*)", out)
    assert funcs, "cuobjdump printed no resource usage"
    seen = set()
    for name, usage in funcs:
        m = re.search(r"SHARED:(\d+)", usage)
        static = max(0, int(m.group(1)) - RESERVED) if m else 0
        for frag, (src, const) in BUDGETS.items():
            if frag in name:
                seen.add(frag)
                dyn = budget(src, const)
                assert static + dyn <= LIMIT, f"{name}: static {static} + dynamic budget {dyn} > {LIMIT}"
        regs = re.search(r"REG:(\d+)", usage)
        assert regs and int(regs.group(1)) <= 255
    assert seen == set(BUDGETS), f"kernels not found in the library: {set(BUDGETS) - seen}"


@pytest.mark.parametrize("conv", model_convs(), ids=lambda c: c[0])
def test_packed_operand_plan_covers_the_bench_models(conv):
    from micronet_b200 import _lib as L
    lib = L.load()
    name, B, Cc, H, W, K, R, st, pad, G = conv
    sh = L.ConvShape(B, Cc, H, W, K, R, R, st, st, pad, pad, 1, 1, G)
    names = "Nt ntiles MT CC chunks nstage smem acc TH TB BW n_mtiles n_items ny".split()
    Tb = min(L.PK_TERMS, L.PK_TERMS_BWD)
    cases = [(0, 1, 1), (1, Tb, 1)]                                  # quantized forward / data gradient with integer weights
    if "res" in name:
        cases += [(0, L.PK_TERMS, L.PK_TERMS), (1, Tb, Tb)]         # the fp32 x fp32 statistics conv of QuantBNFuseConv2d
    for mode, ta, tw in cases:
        plan = (C.c_int32 * 16)()
        assert lib.mnb_pk_conv_plan(C.byref(sh), mode, ta, tw, plan) == 0, (name, mode, ta, tw, lib.mnb_last_error())
        p = dict(zip(names, list(plan)[2:]))
        assert 0 < p["smem"] <= budget("mnb_pk.cu", "kSmemBudget"), (name, p)
        # accumulators of one thread: MT x Nt / 2 registers (two warpgroups of 64 rows each)
        assert p["acc"] == p["MT"] * p["Nt"] and p["acc"] <= 128, (name, p)
        assert p["nstage"] in (2, 4, 8) and p["Nt"] % 16 == 0 and p["Nt"] <= 128 and p["CC"] % 16 == 0, (name, p)
        assert 1 <= p["n_items"] < (1 << 22) and p["n_mtiles"] < (1 << 22), (name, p)           # FastDiv's exact range
        assert p["ny"] == (4 if (mode == 1 and st == 2) else 1), (name, p)                         # stride-2 data gradient: 4 phases
        assert int(lib.mnb_pk_wimage_bytes(C.byref(sh), mode, ta, tw)) >= 16
    P, Q = (H + 2 * pad - R) // st + 1, (W + 2 * pad - R) // st + 1
    if not name.startswith("res224"):            # configs[4] is inference only: no weight gradient at 224 x 224
        assert int(lib.mnb_pk_wgrad_scratch_bytes(C.byref(sh), Tb, 1)) >= 0, name
    # plane sizes: one 16-byte vector per pixel and channel octet and piece
    assert int(lib.mnb_pk_act_bytes(B, Cc, H, W, 1)) == B * ((Cc + 7) // 8) * H * W * 16
    assert int(lib.mnb_pk_act_bytes(B, K, P, Q, Tb)) == Tb * B * ((K + 7) // 8) * P * Q * 16
