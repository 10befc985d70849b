#!/usr/bin/env python
"""Static opcode mix of the level kernels from the built library (cuobjdump, no GPU needed).

Groups SASS opcodes by the pipe that issues them (ncu pipe names): the integer ALU pipe (IADD3, LOP3, SHF,
ISETP, SEL, VIMNMX, PRMT ...), the FMA pipe's integer forms (IMAD and its .IADD / .MOV / .SHL aliases, IDP), memory, shuffles,
control.  Static counts over the whole kernel body (prologue and border code included), so they only indicate the mix of the
hot loop; the executed mix needs an ncu summary (tools/ncu_summary.py)."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
LIB = os.path.join(ROOT, "cineform-sdk_b200", "libcfhd_b200.so")
KERNELS = ["k_fwd_422_tma", "k_fwd_tma<", "k_fwd_plane<0", "k_fwd_plane<2", "k_fwd_plane<3", "k_inv_422_tma<false, false", "k_inv_422_tma<true, false",
           "k_inv_plane<0", "k_inv_plane<2", "k_inv_444<true", "k_sparse_pack", "k_sparse_unpack"]
GROUPS = [
    ("alu", r"^(IADD3|IADD|LOP3|LOP|SHF|SHL|SHR|ISETP|SEL|VIMNMX|IMNMX|PRMT|LEA|VIADD|VABSDIFF|ICMP|BMSK|SGXT|FLO|POPC|BREV|I2I|IABS|ISCADD|PLOP3|P2R|R2P|UIADD3|ULOP3|USHF|UISETP|USEL|ULEA|UPRMT|UMOV|MOV|CS2R|S2R|S2UR|R2UR|UIMAD)"),
    ("fma-int", r"^(IMAD|IDP|IMUL)"),
    ("mem", r"^(LDG|STG|LDS|STS|LDC|LDCU|ULDC|LD|ST|ATOM|ATOMG|RED|CCTL|PREFETCH|UTMALDG|UTMAPF|SYNCS|UBLKCP|LDSM|MEMBAR|FENCE|ERRBAR)"),
    ("shuffle / vote", r"^(SHFL|VOTE|VOTEU|MATCH|REDUX|ELECT)"),
    ("control", r"^(BRA|BRX|EXIT|BSSY|BSYNC|CALL|RET|WARPSYNC|BAR|NOP|NANOSLEEP|YIELD|DEPBAR|BPT|ACQBULK|UCGABAR_ARV|UCGABAR_WAIT|BREAK|BMOV|RPCMOV|KILL|JMP)"),
]


def main():
    text = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in text.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(@!?U?P\d+\s+)?([A-Z0-9_]+)", line)
        if m and cur is not None:
            funcs[cur].append(m.group(2))
    names = subprocess.run(["c++filt"] + list(funcs), capture_output=True, text=True, check=True).stdout.splitlines()
    dem = dict(zip(names, funcs.values()))
    print(f"{'kernel':58s} {'instr':>6s} " + " ".join(f"{g:>14s}" for g, _ in GROUPS) + f" {'other':>7s}")
    for want in KERNELS:
        for name, ops in dem.items():
            if ("cfb::" + want) not in name:
                continue
            cnt, other = collections.Counter(), collections.Counter()
            for op in ops:
                for g, pat in GROUPS:
                    if re.match(pat, op):
                        cnt[g] += 1
                        break
                else:
                    other[op] += 1
            n = len(ops)
            short = name.split("cfb::")[1].split("(")[0]
            print(f"{short[:58]:58s} {n:6d} " + " ".join(f"{cnt[g]:7d} ({100 * cnt[g] // n:2d} %)" for g, _ in GROUPS) +
                  f" {sum(other.values()):7d}" + ("  " + ",".join(f"{k}:{v}" for k, v in other.most_common(4)) if other else ""))


if __name__ == "__main__":
    sys.exit(main())
