"""Per-kernel instruction counts of the built library from `cuobjdump -sass` (no GPU needed).

Used by `tools/sass_summary.py` and `tests/test_sass_cpu.py`.  Hopper mnemonics: HGMMA = wgmma.mma_async; an HGMMA
that carries the `gsb0` operand arms the warpgroup scoreboard that the next WARPGROUP.DEPBAR waits on, so a main loop
that keeps several MMAs in flight issues most of its HGMMAs without it, while a serialized one tags (and waits for)
every single one.  WARPGROUP.ARRIVE = wgmma.fence, WARPGROUP.DEPBAR = wgmma.wait_group, UTMALDG / UTMASTG = TMA
tensor load / store, SYNCS = mbarrier operations."""
from __future__ import annotations

import re
import shutil
import subprocess
from collections import OrderedDict

# counted by the base mnemonic (text before the first '.'), the WARPGROUP ones by their first two parts; HGMMA_WAIT = HGMMA
# with gsb0
WATCH = ("HGMMA", "HGMMA_WAIT", "WARPGROUP.ARRIVE", "WARPGROUP.DEPBAR", "UTMALDG", "UTMASTG", "UTMAPF", "SYNCS",
         "HMMA", "FFMA", "MUFU", "LDG", "STG", "BAR")

_FUNC = re.compile(r"\s*Function : (\S+)")
_INSTR = re.compile(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_.]+)([^;]*);")


def disassemble(path: str) -> str:
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    r = subprocess.run([tool, "-sass", path], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"cuobjdump -sass {path} failed:\n{r.stderr}")
    return r.stdout


def _strip_signature(n: str) -> str:
    """'void vt::(anonymous namespace)::k<128, false>(vt::...)' -> 'vt::k<128, false>'"""
    n = n.replace("(anonymous namespace)::", "").replace("<unnamed>::", "")
    if n.startswith("void "):
        n = n[5:]
    depth = 0
    for i, ch in enumerate(n):
        depth += (ch == "<") - (ch == ">")
        if ch == "(" and depth == 0:
            return n[:i]
    return n


def demangle(names) -> list:
    """kernel names without return type, parameter list and anonymous namespaces (mangled if binutils' c++filt is missing)"""
    names = list(names)
    tool = shutil.which("c++filt")
    if not names or not tool:
        return names
    out = subprocess.run([tool], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    if len(out) != len(names):
        return names
    return [_strip_signature(n) for n in out]


def kernel_counts(sass: str) -> "OrderedDict[str, dict]":
    """mangled kernel name -> {"n": instructions, <WATCH entry>: count, "first": {<entry>: first such line}}"""
    kernels: "OrderedDict[str, dict]" = OrderedDict()
    cur = None
    for line in sass.splitlines():
        m = _FUNC.match(line)
        if m:
            cur = kernels.setdefault(m.group(1), {"n": 0, "first": {}})
            continue
        if cur is None:
            continue
        m = _INSTR.match(line)
        if not m:
            continue
        op, operands = m.group(1), m.group(2)
        cur["n"] += 1
        keys = []
        if op.startswith("WARPGROUP."):
            keys.append(".".join(op.split(".")[:2]))
        else:
            keys.append(op.split(".")[0])
            if keys[0] == "HGMMA" and re.search(r"\bgsb0\b", operands):
                keys.append("HGMMA_WAIT")
        for k in keys:
            if k in WATCH:
                cur[k] = cur.get(k, 0) + 1
                cur["first"].setdefault(k, line.strip())
    return kernels


def serialized_wgmma_kernels(kernels) -> list:
    """kernels that issue HGMMA but every one of them with the scoreboard wait: one MMA in flight at a time"""
    return [name for name, k in kernels.items() if k.get("HGMMA", 0) > 0 and k.get("HGMMA_WAIT", 0) == k["HGMMA"]]
