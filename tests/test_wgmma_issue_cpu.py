"""The compiled tensor-core kernels issue their wgmma back to back: no kernel of the built library waits for each MMA
before issuing the next one.

ptxas inserts `WARPGROUP.DEPBAR` (warpgroup.wait) after an HGMMA / IGMMA whenever the accumulator registers it writes are
used before a wait the program placed itself (ptxas info C7517), e.g. when an accumulator fence pins them in another
register class than the MMA's (`tc::fence_acc` in csrc/mnb_tc.cuh).  Each such wait exposes the full MMA latency; the
narrow-N packed-operand convolutions (m64n16 / m64n32) then run several times above their HBM floor.  A kernel needs one
wait per pipeline stage it retires, plus a few on its edges."""
import re
import shutil
import subprocess

import pytest

MAX_WAITS = 4   # per function; a kernel that waits after every MMA shows one per HGMMA (225 in pk_conv_kernel<*, 16, *>)
# conv_tc_kernel (csrc/mnb_conv_tc_fwd.cu) is serialized for another reason: its wgmma sit in a divergent path, and ptxas
# serializes them around the warpgroup.arrive it inserts there (C7520, "WG.AR in divergent path").  No bench workload runs
# it: the fused NIN-GC graphs run their convolutions on the packed-operand family (pk_conv_kernel).
EXEMPT = ("conv_tc_kernel",)


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_no_wait_after_every_wgmma():
    from micronet_b200 import _lib as L
    out = subprocess.run(["cuobjdump", "-sass", L.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs = {}   # mangled name -> (HGMMA / IGMMA count, WARPGROUP.DEPBAR count)
    for name, body in re.findall(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\Z)", out, re.S):
        mma = len(re.findall(r"\b[HI]GMMA\.", body))
        if mma:
            funcs[name] = (mma, len(re.findall(r"\bWARPGROUP\.DEPBAR\b", body)))
    # every pk_conv_kernel<SEG, NT, I8> instance the library launches is in the dump: bf16 single-product and segmented,
    # and int8 (s32 accumulators in the registers of the float array), at every N tile
    inst = {tuple(map(int, m.groups())) for n in funcs if (m := re.search(r"pk_conv_kernelILb(\d)ELi(\d+)ELb(\d)E", n))}
    for nt in (16, 32, 48, 64, 96, 128):
        assert {(0, nt, 0), (1, nt, 0), (0, nt, 1)} <= inst, nt
    assert any("pk_wgrad_kernel" in n for n in funcs) and any("pk_wgrad_taps_kernel" in n for n in funcs)
    bad = {n: c for n, c in funcs.items() if c[1] > MAX_WAITS and not any(e in n for e in EXEMPT)}
    assert not bad, "functions that wait on their wgmma (HGMMA/IGMMA count, WARPGROUP.DEPBAR count): " + str(bad)
