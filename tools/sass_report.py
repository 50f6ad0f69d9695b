"""Writes profiles/sass_summary.md: per kernel family, the SASS mnemonics that prove what the
kernel does (128-bit peer loads/stores, system-scope release/acquire flags, NVLS multimem ops).
Run on the build box (no GPU needed): ``python tools/sass_report.py``."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "adapcc_b200", "_C", "libadapcc.so")
KEYS = ["LDG.E.NA.128", "STG.E.128", "LDGMC", "STG.E.128.STRONG.SYS", "LDG.E.STRONG.SYS", "STG.E.STRONG.SYS",
        "LDG.E.64.STRONG.SYS", "STG.E.64.STRONG.SYS", "MEMBAR.ALL.SYS", "CCTL.IVALL", "BAR.SYNC", "ATOMG", "REDG",
        "UTCHMMA", "UTCBAR", "UTMALDG", "LDTM", "UTCATOMSWS", "SYNCS"]


def main():
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    names = subprocess.run(["c++filt"], input="\n".join(re.findall(r"Function : (\S+)", sass)), capture_output=True,
                           text=True).stdout.splitlines()
    blocks = re.split(r"\n\s*Function : \S+\n", sass)[1:]
    fam = collections.OrderedDict()
    for name, body in zip(names, blocks):
        key = re.sub(r"<.*", "", name).replace("void ", "").strip()
        d = fam.setdefault(key, {"n": 0, "instr": 0, "c": collections.Counter()})
        d["n"] += 1
        ops = re.findall(r"^\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]+)", body, flags=re.M)
        d["instr"] += len(ops)
        for op in ops:
            for k in KEYS:
                if op.startswith(k):
                    d["c"][k] += 1
    out = ["# SASS evidence (cuobjdump -sass adapcc_b200/_C/libadapcc.so, sm_90a)", "",
           "Counts are summed over all template instantiations of a kernel family. `LDGMC.*` is "
           "`multimem.ld_reduce` (in-switch NVLS reduction), `STG.E.128.STRONG.SYS` on a multicast address is "
           "`multimem.st`; `LDG.E.NA.128` / `STG.E.128` on mapped peer pointers are the 128-bit NVLink loads/stores; "
           "`MEMBAR.ALL.SYS` + `ST*.STRONG.SYS` / `LD*.STRONG.SYS` + `CCTL.IVALL` are the st.release.sys / "
           "ld.acquire.sys flag protocol. `HGMMA` = wgmma.mma_async, `USETMAXREG` = setmaxnreg, `UTMALDG` = TMA tensor "
           "load (`.MULTICAST` = to every CTA of the cluster), `SYNCS` = mbarrier ops.", "",
           "| kernel family | instantiations | SASS instr | " + " | ".join(KEYS) + " |",
           "|---|---|---|" + "---|" * len(KEYS)]
    for k, d in fam.items():
        out.append(f"| `{k}` | {d['n']} | {d['instr']} | " + " | ".join(str(d['c'].get(x, 0)) for x in KEYS) + " |")
    log = os.path.join(ROOT, "adapcc_b200", "_C", "build.log")
    if os.path.exists(log):
        txt = open(log).read()
        regs = re.findall(r"Compiling entry function '(\S+)'.*?Used (\d+) registers.*?\n", txt, flags=re.S)
        spills = re.findall(r"(\d+) bytes spill stores", txt)
        out += ["", f"ptxas: {len(regs)} entry functions, max registers "
                    f"{max((int(r) for _, r in regs), default=0)}, "
                    f"functions with spills: {sum(1 for s in spills if int(s) > 0)}"]
    os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
    with open(os.path.join(ROOT, "profiles", "sass_summary.md"), "w") as f:
        f.write("\n".join(out) + "\n")
    print("\n".join(out[:12]))


if __name__ == "__main__":
    sys.exit(main())
