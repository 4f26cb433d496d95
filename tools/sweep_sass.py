"""Registers, spills and candidate loads in flight of every nn1_kernel instantiation, read from the built library's
SASS: python tools/sweep_sass.py [path/to/libpcu_b200.so]

The k = 1 sweep evaluates a few candidates per trip of its loop.  It only hides the L1/L2 latency of those loads
when all of them are issued before the first instruction that reads one of their results; the register allocator
can quietly serialise them (one 4-register destination reused for both candidates) when the kernel sits at its
launch-bounds register cap.  For each instantiation this prints the registers, the stack frame, the local memory
(spills), the STL/LDL instructions, and how many 128-bit candidate loads (LDG.E.128) the innermost loop that holds
them issues before their first consumer.  Needs cuobjdump, no GPU.
"""
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "point-cloud-utils_b200", "libpcu_b200.so")

_NAME = re.compile(r"nn1_kernelI([fd])NS_9Clouds(Val|Ptr)I[fd]EENS_9Sweeps(Val|Ptr)I[fd]EELb([01])ELb([01])E")
_INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)\s*([^;]*);")
_REG = re.compile(r"\bR(\d+)\b")


def cuobjdump():
    found = shutil.which("cuobjdump")
    if found:
        return found
    cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    return cand if os.path.exists(cand) else None


def label(mangled):
    m = _NAME.search(mangled)
    if not m:
        return None
    t, c, s, out, stats = m.groups()
    return "<%s, Clouds%s, Sweeps%s, kOut=%s, kStats=%s>" % ("float" if t == "f" else "double", c, s,
                                                            "true" if out == "1" else "false",
                                                            "true" if stats == "1" else "false")


def _functions(text, header):
    """{mangled name: body text} for every nn1_kernel section of a cuobjdump listing."""
    out, name, lines = {}, None, []
    for line in text.splitlines():
        m = re.match(r"\s*" + header + r"\s*(\S+?):?\s*$", line)
        if m:
            if name:
                out[name] = "\n".join(lines)
            name, lines = (m.group(1) if "nn1_kernelI" in m.group(1) else None), []
        elif name:
            lines.append(line)
    if name:
        out[name] = "\n".join(lines)
    return out


def _reads(opcode, operands):
    """Registers an instruction reads (the first operand is the destination, except for stores and branches)."""
    parts = [p.strip() for p in operands.split(",")]
    if not opcode.startswith(("ST", "RED", "BRA", "BSSY", "CALL", "RET")):
        parts = parts[1:]
    regs = set()
    for p in parts:
        for m in _REG.finditer(p):
            r = int(m.group(1))
            regs.add(r)
            if p[m.end():].startswith(".64"):
                regs.add(r + 1)
    return regs


def loads_in_flight(sass):
    """(candidate LDG.E.128 issued before their first consumer, instructions in that loop) of one kernel's SASS."""
    insns = []
    for m in _INSN.finditer(sass):
        insns.append((int(m.group(1), 16), m.group(3), m.group(4)))
    loops = []
    for k, (addr, op, args) in enumerate(insns):
        t = re.match(r"\s*(?:U?P\w+\s*,\s*)?0x([0-9a-f]+)", args)
        if op.startswith("BRA") and t and int(t.group(1), 16) < addr:
            start = next(i for i, x in enumerate(insns) if x[0] >= int(t.group(1), 16))
            loops.append((start, k))
    best = None
    for s, e in loops:
        if any(insns[i][1].startswith("LDG.E.128") for i in range(s, e + 1)):
            if best is None or e - s < best[1] - best[0]:
                best = (s, e)
    if best is None:
        return 0, 0
    s, e = best
    body = insns[s:e + 1]
    first = next(i for i, x in enumerate(body) if x[1].startswith("LDG.E.128"))
    pending, issued = set(), 0
    for k in range(len(body)):           # walk the loop once, wrapping at its back edge
        _, op, args = body[(first + k) % len(body)]
        if _reads(op, args) & pending:
            break
        if op.startswith("LDG.E.128"):
            d = int(_REG.search(args).group(1))
            pending |= {d, d + 1, d + 2, d + 3}
            issued += 1
    return issued, len(body)


def report(lib=LIB):
    """One dict per nn1_kernel instantiation: name, regs, stack, local, spill_insns, loads_in_flight, loop_insns."""
    tool = cuobjdump()
    if tool is None:
        raise FileNotFoundError("cuobjdump not found")
    res = subprocess.run([tool, "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    sass = subprocess.run([tool, "-sass", lib], capture_output=True, text=True, check=True).stdout
    usage = {}
    for name, body in _functions(res, "Function").items():
        fields = dict(re.findall(r"(\w+(?:\[\d+\])?):(\d+)", body))
        usage[name] = fields
    rows = []
    for name, body in _functions(sass, r"Function\s*:").items():
        nice = label(name)
        if nice is None:
            continue
        issued, loop = loads_in_flight(body)
        u = usage.get(name, {})
        rows.append(dict(name=nice, mangled=name, regs=int(u.get("REG", -1)), stack=int(u.get("STACK", -1)),
                         local=int(u.get("LOCAL", -1)), spill_insns=len(re.findall(r"\b(?:STL|LDL)\b", body)),
                         loads_in_flight=issued, loop_insns=loop))
    return sorted(rows, key=lambda r: r["name"])


def main():
    lib = sys.argv[1] if len(sys.argv) > 1 else LIB
    rows = report(lib)
    print("%-56s %4s %5s %5s %6s %15s %10s" % ("nn1_kernel instantiation", "regs", "stack", "local", "STL/LDL",
                                                "loads in flight", "loop insns"))
    for r in rows:
        print("%-56s %4d %5d %5d %6d %15d %10d" % (r["name"], r["regs"], r["stack"], r["local"], r["spill_insns"],
                                                   r["loads_in_flight"], r["loop_insns"]))


if __name__ == "__main__":
    main()
