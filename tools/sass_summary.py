"""SASS evidence: per kernel of libvidtok_b200.so (sm_90a), the count of tensor-core / TMA / barrier instructions.
  python tools/sass_summary.py OUT_DIR [LIB]  ->  OUT_DIR/sass_summary.txt
LIB defaults to the in-tree vidtok_b200/libvidtok_b200.so.  Mnemonics (vidtok_b200/sass.py): HGMMA = wgmma.mma_async,
HGMMA_WAIT = those of them that carry the gsb0 scoreboard (a pipelined main loop has fewer of these than HGMMAs),
WARPGROUP.ARRIVE / DEPBAR = wgmma.fence / wait_group, UTMALDG / UTMASTG = TMA tensor load / store, SYNCS = mbarrier."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from vidtok_b200 import sass  # noqa: E402


def main():
    if len(sys.argv) < 2:
        sys.exit(__doc__)
    out_dir = sys.argv[1]
    lib = sys.argv[2] if len(sys.argv) > 2 else os.path.join(ROOT, "vidtok_b200", "libvidtok_b200.so")
    kernels = sass.kernel_counts(sass.disassemble(lib))
    serialized = set(sass.serialized_wgmma_kernels(kernels))
    os.makedirs(out_dir, exist_ok=True)
    out = os.path.join(out_dir, "sass_summary.txt")
    with open(out, "w") as f:
        f.write(f"# cuobjdump -sass {os.path.basename(lib)} (sm_90a), instruction counts per kernel\n")
        f.write("# HGMMA = wgmma.mma_async, HGMMA_WAIT = HGMMA with the gsb0 scoreboard, WARPGROUP.ARRIVE/DEPBAR = wgmma fence / "
                "wait_group,\n# UTMALDG/UTMASTG = TMA tensor load/store, SYNCS = mbarrier.\n\n")
        for (mang, k), name in zip(kernels.items(), sass.demangle(kernels)):
            counts = "  ".join(f"{w}={k[w]}" for w in sass.WATCH if w in k)
            f.write(f"{name}\n    {k['n']} instructions   {counts}\n")
            if mang in serialized:
                f.write("    SERIALIZED: every HGMMA waits for the previous one\n")
            for w in ("HGMMA", "UTMALDG", "UTMASTG"):
                if w in k["first"]:
                    f.write(f"      e.g. {k['first'][w]}\n")
            f.write("\n")
    print("wrote", out, len(kernels), "kernels,", len(serialized), "with serialized wgmma")


if __name__ == "__main__":
    main()
