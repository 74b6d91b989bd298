"""SASS evidence: per kernel family the instruction mix of the built library and the
Hopper-specific mnemonics (UBLKCP = cp.async.bulk, UTMALDG = TMA tensor tile, SYNCS = mbarrier,
STAS = st.async to a peer CTA's shared memory, UCGABAR = cluster barrier, MUFU.RCP = the hoisted
reciprocals of the stereo SOR).  No GPU needed:
    python tools/sass_dump.py > sass_summary.txt
    python tools/sass_dump.py --full sor_wave_kernelILi2ELi64ELi1ELi0 > sass_sor_flow.txt"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "of_dis_b200", "lib", "libofdis_b200.so")
KEY = ["UBLKCP", "UTMALDG", "SYNCS", "STAS", "UCGABAR", "LDGSTS", "LDGDEPBAR", "DEPBAR", "CREDUX", "ACQBULK", "MUFU.RCP", "MUFU.RSQ", "FCHK", "CALL", "BAR.SYNC", "LDS", "STS",
       "LDG", "STG", "SHFL", "VOTE", "FFMA", "FMUL", "FADD", "FSEL", "MEMBAR", "FENCE", "CCTL"]


def functions():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    cur, body = None, {}
    for ln in out.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            body[cur] = []
        elif cur and re.match(r"\s+/\*[0-9a-f]{4,}\*/", ln):
            body[cur].append(ln)
    return body


def opcode(ln):
    t = re.sub(r"/\*.*?\*/", "", ln).strip().rstrip(";").split()
    if not t:
        return None
    if t[0].startswith("@"):
        t = t[1:]
    return t[0] if t else None


if __name__ == "__main__":
    body = functions()
    if len(sys.argv) > 2 and sys.argv[1] == "--full":
        for name, lines in body.items():
            if sys.argv[2] in name:
                print("// %s (%d instructions)" % (name, len(lines)))
                print("\n".join(re.sub(r"\s*/\* 0x[0-9a-f]+ \*/\s*$", "", l) for l in lines))
        sys.exit(0)
    print("# cuobjdump -sass of_dis_b200/lib/libofdis_b200.so : instructions per kernel and selected mnemonics")
    for name in sorted(body):
        ops = collections.Counter()
        for ln in body[name]:
            op = opcode(ln)
            if op:
                ops[op] += 1
        short = re.sub(r"^_ZN5ofdis\d+_GLOBAL__N__[0-9a-f]+_\d+_[a-z_]+_cu_[0-9a-f]+\d*", "", name)
        sel = {k: sum(v for o, v in ops.items() if o.startswith(k)) for k in KEY}
        print("%-70s %5d instr  %s" % (short[:70], sum(ops.values()), " ".join("%s=%d" % (k, v) for k, v in sel.items() if v)))
