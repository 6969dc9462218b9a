"""SASS of the ray-BVH node visit (trace.cuh:node_test) in every traversal kernel: its load batches and its instruction mix.

    python scripts/sass_node_visit.py [LIB]          LIB defaults to rmcl_b200/lib/librmcl_b200.so (build it first); CPU only

A visit starts at the 64-bit node address (IMAD.WIDE.U32 by the node size, 0xe0) and ends at the first multiply by 7 (spread3x: leaf-child
hit bits to triangle bits) after its 13th load.  Inside it, the 13 node loads are LDG.E.128 from that address.  A load BATCH is
a run of loads with no instruction between them that reads the data of an earlier load of the same visit: every load of a batch is
in flight before the visit waits on any of them.  An L1 miss of a load in batch n cannot overlap with the misses of batch n - 1, so
the batch count bounds the dependent trips to L2 / DRAM of a visit whose node is not in L1.  Each load is shown by its immediate
offset (+0x10: quad b of a plane array, +0xc0: the header quad; the plane arrays themselves are per-ray register offsets).
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNELS = ("k_rcc_find", "k_intersect", "k_rcc_fused_batch", "k_pf_update", "k_pf_motion", "k_pf_surface", "k_pf_recovery_inject")
INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)\s*(.*?)\s*;")
REG = re.compile(r"\bR(\d+)\b")
MIX = ("LDG", "FFMA", "FMNMX", "FSETP", "VIMNMX3", "VIMNMX", "IMNMX", "ISETP", "LOP3", "SHF", "SEL", "PRMT", "IADD3", "IMAD", "LEA", "MOV")


def functions(lib):
    out = subprocess.run(["cuobjdump", "-sass", lib], check=True, capture_output=True, text=True).stdout
    name, body = None, []
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            if name:
                yield name, body
            name, body = m.group(1), []
            continue
        m = INSN.search(line)
        if m and name:
            body.append((m.group(3), m.group(4)))
    if name:
        yield name, body


def demangled(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return dict(zip(names, out)) if len(out) == len(names) else {n: n for n in names}


def regs(op, text):
    """(written, read) register numbers of one instruction; 64- and 128-bit operands cover 2 / 4 registers."""
    parts = [p.strip() for p in text.split(",")]
    width = 4 if ".128" in op else 2 if ".64" in op else 1
    written, read = set(), set()
    stores = op.startswith(("ST", "RED", "ATOM", "BRA", "ISETP", "FSETP", "BAR"))
    for k, p in enumerate(parts):
        for m in REG.finditer(p):
            r = int(m.group(1))
            span = 2 if ".64" in p[m.end():m.end() + 3] else 1
            if k == 0 and not stores and "[" not in p:
                written.update(range(r, r + (width if op.startswith("LDG") else (2 if ".WIDE" in op else 1))))
            else:
                read.update(range(r, r + span))
    return written, read


def visits(body):
    """[(start, end)] instruction ranges of the node visits in one function."""
    out = []
    for i, (op, text) in enumerate(body):
        if op.startswith("IMAD.WIDE.U32") and re.search(r",\s*0xe0\b", text):
            loads = 0
            for j in range(i + 1, min(i + 400, len(body))):
                loads += body[j][0].startswith("LDG.E.128")
                if loads >= 13 and body[j][0] == "IMAD" and re.search(r",\s*0x7,\s*RZ$", body[j][1]):
                    out.append((i, j + 1))
                    break
    return out


def analyse(body, a, b):
    batches, cur, pending, consumed = [], [], set(), False
    mix = collections.Counter()
    for op, text in body[a:b]:
        w, r = regs(op, text)
        base = op.split(".")[0]
        mix[base if base in MIX else "other"] += 1
        if op.startswith("LDG.E.128") or op.startswith("CCTL.E.PF"):
            if consumed and cur:
                batches.append(cur)
                cur, consumed = [], False
            m = re.search(r"\+(0x[0-9a-f]+)\]", text)
            cur.append("+" + (m.group(1) if m else "0"))
            pending |= w
            continue
        if r & pending:
            consumed = True
        pending -= w
    if cur:
        batches.append(cur)
    return b - a, batches, mix


def main():
    lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "rmcl_b200", "lib", "librmcl_b200.so")
    funs = [(n, body) for n, body in functions(lib) if any(k in n for k in KERNELS)]
    names = demangled([n for n, _ in funs])
    for n, body in sorted(funs, key=lambda x: names[x[0]]):
        vs = visits(body)
        print("%s: %d node visit(s)" % (names[n].split("(")[0] + ("<" + names[n].split("<", 1)[1].split(">")[0] + ">" if "<" in names[n].split("(")[0] else ""), len(vs)))
        for a, b in vs:
            n_insn, batches, mix = analyse(body, a, b)
            kind = "int" if mix["VIMNMX3"] else "float"
            print("  %s reduction, %d instructions, %d load batch(es): %s" % (kind, n_insn, len(batches), " | ".join(" ".join(x) for x in batches)))
            print("    " + " ".join("%s %d" % (k, mix[k]) for k in MIX + ("other",) if mix[k]))


if __name__ == "__main__":
    main()
