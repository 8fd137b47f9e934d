#!/usr/bin/env python3
"""Per-pipe instruction mix of a kernel's main loop, from the SASS of a built library (no GPU needed).

    python scripts/sass_pipe_mix.py cimba_b200/lib/libcimba_b200.so mm1_kernelILb0 [--list]
        [--exclude START-END,...] [--steps N]

The loop = the backward branch with the largest span (as scripts/sass_loop_stats.py); every instruction inside it is counted,
rare blocks included, unless --exclude names address ranges (hex, both ends included, as --list prints them) to leave out:
the rare blocks, so that what remains is the path most iterations take.  --steps N also prints the counts divided by N, for
a loop whose body runs N event steps.  Pipes as ncu's sm__inst_executed_pipe_* names them: alu (integer add / logic / shift / compare /
select - half rate), fma (IMAD*, FP32), fp64, xu (conversions, MUFU, POPC), lsu (shared / global / local memory), cbu (branches,
convergence barriers), uniform (U* datapath)."""
import collections
import re
import subprocess
import sys

PIPE = {
    "alu": "LOP3 SHF IADD3 ISETP SEL FSEL PRMT LEA VIADD VIMNMX PLOP3 IABS FSETP MOV FMNMX LOP BMSK SGXT FLO BREV IADD ISCADD VABSDIFF R2P P2R CS2R".split(),
    "fma": "IMAD FFMA FMUL FADD HFMA2 IDP IMUL".split(),
    "fp64": "DADD DMUL DFMA DSETP".split(),
    "xu": "I2F F2I F2F MUFU POPC I2I FRND".split(),
    "lsu": "LDS STS LDG STG LDL STL LD ST ATOMS ATOMG RED REDG ATOM LDSM MEMBAR LDC".split(),
    "cbu": "BRA BSSY BSYNC EXIT CALL RET WARPSYNC BREAK BRX JMP NANOSLEEP YIELD BPT ENDCOLLECTIVE".split(),
    "warp": "VOTE SHFL MATCH REDUX S2R NOP ELECT".split(),
}
OF = {op: pipe for pipe, ops in PIPE.items() for op in ops}


def loop_of(so, pat):
    txt = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    blocks = re.split(r"\n\s*Function : ", txt)
    body = [b for b in blocks if pat in b.split("\n", 1)[0]][0]
    ins = []
    for l in body.splitlines():
        m = re.match(r"\s*/\*([0-9a-f]{4,6})\*/\s+(.*?);", l)
        if m:
            ins.append((int(m.group(1), 16), m.group(2).strip()))
    back = []
    for a, t in ins:
        m = re.search(r"\bBRA\b.*?0x([0-9a-f]+)", t)
        if m and int(m.group(1), 16) < a:
            back.append((a - int(m.group(1), 16), int(m.group(1), 16), a))
    _, start, end = max(back)
    return [(a, t) for a, t in ins if start <= a <= end]


def option(name, default=None):
    return sys.argv[sys.argv.index(name) + 1] if name in sys.argv else default


def main():
    so, pat = sys.argv[1], sys.argv[2]
    loop = loop_of(so, pat)
    excluded = []
    for r in filter(None, option("--exclude", "").split(",")):
        lo, hi = (int(x, 16) for x in r.split("-"))
        excluded.append((lo, hi))
    full = len(loop)
    loop = [(a, t) for a, t in loop if not any(lo <= a <= hi for lo, hi in excluded)]
    steps = int(option("--steps", "1"))
    mix, ops = collections.Counter(), collections.Counter()
    for _, t in loop:
        op = re.sub(r"^@!?U?P\d+\s+", "", t).split()[0].split(".")[0]
        pipe = "uniform" if op.startswith("U") and op not in ("UNKNOWN",) else OF.get(op, "other")
        mix[pipe] += 1
        ops[(pipe, op)] += 1
    n = len(loop)
    print(f"{pat}: loop 0x{loop[0][0]:x}..0x{loop[-1][0]:x}, {n} instructions"
          + (f" ({full - n} in {len(excluded)} excluded ranges left out)" if excluded else ""))
    for pipe, c in mix.most_common():
        detail = ", ".join(f"{op} {k}" for (p, op), k in sorted(ops.items(), key=lambda x: -x[1]) if p == pipe)
        print(f"  {pipe:8s} {c:4d} ({100 * c / n:4.1f} %)" + (f"  {c / steps:6.1f} per step" if steps > 1 else "") + f"  {detail}")
    if steps > 1:
        print(f"  issued   {n:4d}            {n / steps:6.1f} per step")
    if "--list" in sys.argv:
        for a, t in loop:
            print(f"    {a:05x}  {t}")


if __name__ == "__main__":
    main()
