"""Compiler-output checks of the tensor-core kernels (cuobjdump cross-disassembles the sm_90a library, no GPU needed).

Every kernel that issues wgmma must keep more than one MMA in flight: a main loop in which each HGMMA carries the
scoreboard wait runs the tensor pipe at a fraction of its rate while computing the same numbers, so nothing but this
check notices it."""
import os

from vidtok_b200 import build, sass


def _kernels():
    lib = build.build()
    assert os.path.exists(lib)
    return sass.kernel_counts(sass.disassemble(lib))


def test_wgmma_main_loops_are_pipelined():
    kernels = _kernels()
    hg = {name: k for name, k in kernels.items() if k.get("HGMMA", 0) > 0}
    # the bf16 and split-fp16 convolutions (mangled conv_tc_kernel<BN, split>), the fused temporal block and the stem
    # all run on wgmma
    for want in ("conv_tc_kernelILi128ELb0E", "conv_tc_kernelILi256ELb0E", "conv_tc_kernelILi128ELb1E", "tblock_tc_kernel",
                 "conv_stem_kernel"):
        assert any(want in n for n in hg), f"no HGMMA in {want}"
    names = dict(zip(hg, sass.demangle(hg)))
    serialized = sass.serialized_wgmma_kernels(hg)
    detail = [f"{names[n]}: {hg[n]['HGMMA']} HGMMA, all with a wait" for n in serialized]
    assert not serialized, "wgmma issued one at a time:\n  " + "\n  ".join(detail)
