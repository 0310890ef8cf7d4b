#!/usr/bin/env python3
"""Static (no-GPU) evidence for every kernel in libglim_b200.so: ptxas resources (registers, spills, shared memory) from the
build logs and selected SASS mnemonic counts from `cuobjdump -sass`.  Output: markdown on stdout.
Measurement plumbing; nothing here is imported by the product."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "glim_b200", "csrc", "build")
SO = os.path.join(ROOT, "glim_b200", "libglim_b200.so")

# mnemonic prefixes worth counting: what proves (or disproves) the claims DESIGN.md makes about each kernel
WATCH = [
    ("LDG.E.128", r"\bLDG\.E\.128"),            # float4 / 16-byte gathers
    ("LDG (all)", r"\bLDG\."),
    ("LDS", r"\bLDS"),
    ("STS", r"\bSTS"),
    ("STG.E.128", r"\bSTG\.E\.128"),
    ("ATOMG.ADD.F64", r"\bATOMG\.E\.ADD\.F64"),  # fp64 reductions into the factor accumulators (result unused: RZ)
    ("ATOMG.ADD.F32", r"\bATOMG\.E\.ADD\.F32"),  # fp32 adds into a local pair slab (gb_sweep_set_slab; not used with a peer slab)
    ("ATOMG (int)", r"\bATOMG\.E\.(ADD|MIN|MAX|CAS|EXCH)(\.64)?\.STRONG"),
    ("SHFL", r"\bSHFL\."),
    ("VOTE/MATCH", r"\bVOTE\.|\bMATCH\."),
    ("MEMBAR.ALL.GPU", r"\bMEMBAR\.ALL\.GPU"),
    ("MEMBAR.SC / .SYS", r"\bMEMBAR\.(SC|ALL\.SYS)"),
    ("CCTL.IVALL", r"\bCCTL\.IVALL"),
    ("BAR.SYNC", r"\bBAR\.SYNC"),
    ("DFMA/DMUL/DADD", r"\bD(FMA|MUL|ADD)\b"),
    ("FFMA", r"\bFFMA\b"),
    ("MUFU", r"\bMUFU\."),
    ("STL/LDL (local)", r"\b(STL|LDL)\b"),
]


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), text=True, capture_output=True).stdout.splitlines()
    res = {}
    for n, d in zip(names, out):
        d = re.sub(r"\(anonymous namespace\)::", "", d)
        d = re.sub(r"_GLOBAL__N__[0-9a-f_]+_cu_[0-9a-f]+::", "", d)
        d = re.sub(r"^void ", "", d)
        d = re.sub(r"\(.*$", "", d)
        res[n] = d
    return res


def ptxas_resources():
    rows = {}
    for log in sorted(os.listdir(BUILD)):
        if not log.endswith(".ptxas.log"):
            continue
        txt = open(os.path.join(BUILD, log)).read()
        for m in re.finditer(
            r"Compiling entry function '([^']+)' for 'sm_90a'\n.*?\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n"
            r"ptxas info\s+: Used (\d+) registers(?:, used (\d+) barriers)?(?:, (\d+) bytes cumulative stack size)?(?:, (\d+) bytes smem)?",
            txt,
        ):
            rows[m.group(1)] = dict(file=log.replace(".ptxas.log", ".cu"), stack=int(m.group(2)), sst=int(m.group(3)), sld=int(m.group(4)), regs=int(m.group(5)), smem=int(m.group(8) or 0))
    return rows


def sass_counts():
    txt = subprocess.run(["cuobjdump", "-sass", SO], text=True, capture_output=True).stdout
    counts = {}
    cur = None
    for line in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            counts[cur] = collections.Counter()
            continue
        if cur is None or "/*" not in line:
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if not m:
            continue
        ins = m.group(1)
        counts[cur]["(instructions)"] += 1
        for label, pat in WATCH:
            if re.search(pat, ins):
                counts[cur][label] += 1
    return counts


def keep(name):
    """our kernels only (CUB's sort / scan / reduce kernels are toolkit code); of the k-NN kernels' K instantiations only K = 10
    (config_preprocess.json:33) and K = 20"""
    if "cub::" in name or not name.startswith("k_"):
        return False
    m = re.match(r"k_knn_\w+<(\d+)>", name)
    return not m or m.group(1) in ("10", "20")


def main():
    res = ptxas_resources()
    sass = sass_counts()
    names = sorted(set(res) | set(sass))
    dm = demangle(names)
    print("# Static resources and SASS mnemonics of every kernel in `libglim_b200.so` (sm_90a, nvcc 12.9, `-O3 -lineinfo`)")
    print()
    print("Produced without a GPU by `python scripts/static_report.py` from `glim_b200/csrc/build/*.ptxas.log` (`-Xptxas -v`) and")
    print("`cuobjdump -sass glim_b200/libglim_b200.so`.  Template arguments of the sweep kernels: `k_vgicp_sweep3<MODE, PEER, SV>`,")
    print("`k_vgicp_sweep5<MODE, PEER>`; MODE 0 = linearize, 1 = error;")
    print("PEER = finished pair rows are pushed to a (peer) slab; SV = surface validation compiled in.")
    print()
    print("## Resources (ptxas)")
    print()
    print("| kernel | file | regs | static smem B | stack B | spill st / ld B |")
    print("|---|---|---|---|---|---|")
    for n in sorted(res, key=lambda k: (res[k]["file"], dm[k])):
        r = res[n]
        if not keep(dm[n]):
            continue
        print(f"| `{dm[n]}` | {r['file']} | {r['regs']} | {r['smem']} | {r['stack']} | {r['sst']} / {r['sld']} |")
    print()
    print("## SASS mnemonic counts (static instruction counts, not executed counts)")
    print()
    labels = ["(instructions)"] + [w[0] for w in WATCH]
    print("| kernel | " + " | ".join(labels) + " |")
    print("|---|" + "---|" * len(labels))
    for n in sorted(sass, key=lambda k: dm.get(k, k)):
        if not keep(dm.get(n, n)):
            continue
        c = sass[n]
        print(f"| `{dm.get(n, n)}` | " + " | ".join(str(c.get(l, 0)) for l in labels) + " |")
    print()
    print("Reading guide (source lines from `nvdisasm -g` of the same cubin):")
    print("* the committed hot kernels (`k_vgicp_sweep3<0,*,*>`, `k_vgicp_sweep5<0,*>`) gather with `LDG.E.128`, reduce with `SHFL` and one")
    print("  `ATOMG.E.ADD.F64` per lane (the transposing reduce-scatter leaves one of the 29 sums in each lane; result unused);")
    print("* every `MEMBAR.ALL.GPU` is half of an `atom.add.release.gpu` ticket (`ticket_release`, gb_kernels_vgicp.cu:221) or of the")
    print("  `fence.acq_rel.gpu` (`fence_acquire`, :226) that only the warp drawing a factor's / pair's LAST ticket executes; the two")
    print("  `CCTL.IVALL` (L1 invalidate) belong to that acquire, i.e. once per factor, not once per item; there is no `MEMBAR.SC`")
    print("  (`__threadfence()`) in the sweep kernels -- `MEMBAR.ALL.SYS` appears only in the two exchange kernels (`__threadfence_system`);")
    print("* local-memory instructions of sweep3 / sweep5 are the call frame of the `__noinline__` epilogue (`factor_epilogue`): the")
    print("  argument stores ahead of its two calls and one load inside it; `acc[32]` stays in registers through the item reduction.")


if __name__ == "__main__":
    sys.exit(main())
