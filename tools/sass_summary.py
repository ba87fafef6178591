#!/usr/bin/env python
"""What the shipped cubin contains, per kernel: code size, registers / stack / spills (ptxas), and the mnemonics that show how
bytes move - 128-bit global loads / stores, TMA bulk copies and their mbarrier traffic, shuffles, local-memory (stack) accesses,
tensor-core ops (none: this path has no FLOPs).  Needs no GPU.

    python tools/sass_summary.py > sass.md
"""
import collections
import os
import re
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(REPO, "min-tfs-client_b200", "lib", "libb200tfs.so")
CSRC = os.path.join(REPO, "min-tfs-client_b200", "csrc")

PATTERNS = collections.OrderedDict([
    ("LDG.E.128 (128-bit global loads)", r"\bLDG\.E(\.[A-Z0-9_]+)*\.128\b"),
    ("STG.E.128 (128-bit global stores)", r"\bSTG\.E(\.[A-Z0-9_]+)*\.128\b"),
    ("LDG other widths", r"\bLDG\.E(?!(\.[A-Z0-9_]+)*\.128)"),
    ("STG other widths", r"\bSTG\.E(?!(\.[A-Z0-9_]+)*\.128)"),
    ("UBLKCP (TMA bulk copy global->shared)", r"\bUBLKCP\b"),
    ("SYNCS (mbarrier arrive / try_wait)", r"\bSYNCS\b"),
    ("LDS.128 / STS.128", r"\b(LDS|STS)(\.[A-Z0-9_]+)*\.128\b"),
    ("SHFL (warp shuffles)", r"\bSHFL\b"),
    ("SHF (funnel shifts)", r"\bSHF\b"),
    ("LDL / STL (local memory = stack)", r"\b(LDL|STL)\b"),
    ("LDC (parameter / constant loads)", r"\bLDC\b"),
    ("ATOM / RED (atomics)", r"\b(ATOMG|ATOM|RED|ATOMS)\b"),
    ("BAR (CTA barriers)", r"\bBAR\b"),
    ("tensor core (HMMA / UTC*MMA / tcgen05)", r"\b(HMMA|IMMA|UTCHMMA|UTCQMMA|UTCIMMA|UTCMMA)\b"),
])


def sass():
    out = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True).stdout
    kernels, name = collections.OrderedDict(), None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            kernels[name] = []
            continue
        if name and re.match(r"\s+/\*[0-9a-f]{4,}\*/", line):
            kernels[name].append(line)
    return kernels


def ptxas():
    flags = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-Xptxas", "-v", "-c",
             os.path.join(CSRC, "kernels.cu"), "-o", "/tmp/_sass_summary.o"]
    err = subprocess.run(["nvcc"] + flags, capture_output=True, text=True).stderr
    info, cur = {}, None
    for line in err.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            info[cur] = {}
            continue
        if cur:
            m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
            if m:
                info[cur].update(stack=int(m.group(1)), spill_st=int(m.group(2)), spill_ld=int(m.group(3)))
            m = re.search(r"Used (\d+) registers", line)
            if m:
                info[cur]["regs"] = int(m.group(1))
                m2 = re.search(r"(\d+) bytes smem", line)
                info[cur]["smem"] = int(m2.group(1)) if m2 else 0
    return info


def demangle(n):
    m = re.match(r"_ZN7b200tfs(\d+)", n)
    return n[len(m.group(0)): len(m.group(0)) + int(m.group(1))] if m else n


def main():
    ks, info = sass(), ptxas()
    print("# SASS of the shipped library (`min-tfs-client_b200/lib/libb200tfs.so`, sm_90a) - `python tools/sass_summary.py`\n")
    print("Per kernel: instructions (x 16 B = code size), registers / stack / spill bytes / static shared memory as ptxas reports them, and how "
          "many instructions of each kind the cubin holds (static counts, not executed counts).\n")
    print("| kernel | SASS instr | code KB | regs | stack B | spill st/ld B | smem B |")
    print("|---|---|---|---|---|---|---|")
    for n, lines in ks.items():
        i = info.get(n, {})
        print(f"| `{demangle(n)}` | {len(lines)} | {len(lines) * 16 // 1024} | {i.get('regs', '?')} | {i.get('stack', '?')} | "
              f"{i.get('spill_st', '?')}/{i.get('spill_ld', '?')} | {i.get('smem', '?')} |")
    print()
    heads = list(PATTERNS)
    print("| kernel | " + " | ".join(h.split(" (")[0] for h in heads) + " |")
    print("|---|" + "---|" * len(heads))
    for n, lines in ks.items():
        text = "\n".join(lines)
        print(f"| `{demangle(n)}` | " + " | ".join(str(len(re.findall(p, text))) for p in PATTERNS.values()) + " |")
    print("\nLegend: " + "; ".join(heads) + ".")
    print("\nReading guide: the payload paths (`move_kernel*`, `decode_fused*`) move bytes with `LDG.E.128` / `STG.E.128` only; the batch decode "
          "kernel additionally fetches its tiles with TMA bulk copies (`UBLKCP` + `SYNCS` mbarrier traffic).  `LDL` / `STL` belong to the cold tag "
          "walk (`fused_slow_path`: its group stack and chunk sort live in local memory) - the template path of the decode kernels touches none. "
          "No tensor-core instruction anywhere: the path has zero FLOPs.")


if __name__ == "__main__":
    main()
