"""SASS census of the two-row skewed fill kernel's cell loops (csrc/convex_fill.cu). CPU only: no GPU is needed.

Compiles convex_fill.cu for sm_90a with the Makefile's NVFLAGS into a cubin, disassembles it with cuobjdump, and for
convex_fill_rf2_kernel<RAW, PERSIST=false, SKEW=true> (RAW = false, the default scoring, and RAW = true) finds the
innermost loops of fill_group2: the only loops whose body holds 16 SHFL.IDX (four unrolled steps of four shuffles)
and no branch but the loop's own. The one that loads reference bytes (LDG, SELF_REF) is the masked loop, the other the
all-active one. For each it prints the instructions per 4 steps (8 cells per lane) by pipe and by opcode, and the
kernel's registers and spills from ptxas -v.

    python scripts/fill_sass.py [--opcodes] [--json FILE] [--nvcc PATH] [--src FILE]

The pipe of an opcode is what the Hopper tuning guide and the instruction throughput table give: the half-rate ALU
pipe (compares, selects, min/max, logic, shifts, integer adds), the FMA pipe (FADD/FMUL/FFMA and every IMAD form,
IMAD.MOV included), MIO (shuffles, shared and global memory), other (branches, CS2R, constant loads, and the sm_90
VIADD / VIADDMNMX, whose pipe is not documented).
"""
import argparse
import collections
import json
import os
import re
import shlex
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "ngmlr_b200", "csrc")

ALU = {"FSETP", "FMNMX", "SEL", "FSEL", "PLOP3", "ISETP", "FSET", "LOP3", "SHF", "IADD3", "LEA", "IMNMX", "PRMT",
       "MOV", "P2R", "R2P", "IABS", "FLO", "POPC", "BMSK", "VIMNMX"}
FMA = {"FADD", "FMUL", "FFMA", "IMAD", "IMUL", "HFMA2", "HADD2", "HMUL2", "IDP", "IMNMX3"}
MIO = {"SHFL", "LDS", "STS", "LDG", "STG", "LD", "ST", "ATOMS", "ATOMG", "RED", "LDSM"}


def pipe(op):
    base = op.split(".")[0]
    if base in ALU:
        return "alu"
    if base in FMA:
        return "fma"
    if base in MIO:
        return "mio"
    return "other"


def nvflags():
    """NVFLAGS of the Makefile with $(ARCH) expanded."""
    vars_ = {}
    with open(os.path.join(CSRC, "Makefile")) as f:
        for line in f:
            m = re.match(r"^(\w+)\s*[:?]?=\s*(.*)$", line.strip())
            if m:
                vars_[m.group(1)] = m.group(2)
    flags = vars_["NVFLAGS"]
    for k, v in vars_.items():
        flags = flags.replace(f"$({k})", v)
    return shlex.split(flags)


def compile_cubin(nvcc, src, out_dir):
    cubin = os.path.join(out_dir, "convex_fill.cubin")
    flags = [f for f in nvflags() if f not in ("-c",)]
    cmd = [nvcc] + flags + ["-cubin", src, "-o", cubin]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=CSRC)
    if r.returncode != 0:
        raise SystemExit(f"nvcc failed:\n{' '.join(cmd)}\n{r.stdout}{r.stderr}")
    return cubin, r.stdout + r.stderr


def ptxas_info(log):
    """mangled kernel name -> {registers, spill_stores, spill_loads, stack}"""
    info, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            info[cur] = {}
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            info[cur].update(stack=int(m.group(1)), spill_stores=int(m.group(2)), spill_loads=int(m.group(3)))
        m = re.search(r"Used (\d+) registers", line)
        if m and cur:
            info[cur]["registers"] = int(m.group(1))
    return info


def functions(cubin):
    """mangled name -> [(address, predicate, opcode, operands)]"""
    r = subprocess.run(["cuobjdump", "-sass", cubin], capture_output=True, text=True, check=True)
    funcs, cur = {}, None
    for line in r.stdout.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(@!?U?P\w+\s+)?(\S+)\s*(.*?)\s*;", line)
        if m and cur is not None:
            cur.append((int(m.group(1), 16), (m.group(2) or "").strip(), m.group(3), m.group(4)))
    return funcs


def cell_loops(ins):
    """(kind, body) of every innermost loop with 16 SHFL.IDX and a single branch"""
    at = {a: i for i, (a, *_rest) in enumerate(ins)}
    loops = []
    for i, (a, _p, op, args) in enumerate(ins):
        if op.split(".")[0] != "BRA":
            continue
        m = re.search(r"0x([0-9a-f]+)\s*$", args)
        if not m or int(m.group(1), 16) >= a:
            continue
        body = ins[at[int(m.group(1), 16)]:i + 1]
        nshfl = sum(x[2].startswith("SHFL.IDX") for x in body)
        nbra = sum(x[2].split(".")[0] == "BRA" for x in body)
        if nshfl == 16 and nbra == 1:
            kind = "masked" if any(x[2].startswith("LDG") for x in body) else "all-active"
            loops.append((kind, body))
    return loops


def census(body, steps):
    scale = 4.0 / steps
    by_op = collections.Counter(op for _a, _p, op, _x in body)
    by_pipe = collections.Counter(pipe(op) for _a, _p, op, _x in body)
    f = lambda n: round(n * scale, 2)
    return {"instructions": f(len(body)), "pipes": {k: f(by_pipe.get(k, 0)) for k in ("alu", "fma", "mio", "other")},
            "alu_issue_cycles": f(2 * by_pipe.get("alu", 0)),
            "opcodes": {k: f(v) for k, v in sorted(by_op.items(), key=lambda kv: (-kv[1], kv[0]))}}


def kernel_name(raw):
    return f"convex_fill_rf2_kernelILb{int(raw)}ELb0ELb1EE"


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--nvcc", default=os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"))
    ap.add_argument("--src", default=os.path.join(CSRC, "convex_fill.cu"))
    ap.add_argument("--opcodes", action="store_true", help="also list every opcode per 4 steps")
    ap.add_argument("--json", default=None, help="write the census as JSON")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        cubin, log = compile_cubin(args.nvcc, os.path.abspath(args.src), tmp)
        funcs = functions(cubin)
    regs = ptxas_info(log)
    out = {}
    for raw in (False, True):
        key = kernel_name(raw)
        name = next((n for n in funcs if key in n), None)
        if name is None:
            raise SystemExit(f"no function matching {key} in the cubin")
        label = f"<RAW={'true' if raw else 'false'}, PERSIST=false, SKEW=true>"
        rinfo = regs.get(name, {})
        out[label] = {"registers": rinfo.get("registers"), "spill_stores": rinfo.get("spill_stores"),
                      "spill_loads": rinfo.get("spill_loads"), "stack": rinfo.get("stack"), "loops": {}}
        loops = cell_loops(funcs[name])
        kinds = [k for k, _ in loops]
        if sorted(kinds) != ["all-active", "masked"]:
            raise SystemExit(f"{label}: expected one all-active and one masked cell loop, found {kinds}")
        print(f"{label}: {rinfo.get('registers')} registers, {rinfo.get('spill_stores')} B spill stores, "
              f"{rinfo.get('spill_loads')} B spill loads, {rinfo.get('stack')} B stack")
        for kind, body in sorted(loops, key=lambda kb: kb[0] != "all-active"):
            steps = sum(x[2].startswith("SHFL.IDX") for x in body) // 4
            c = census(body, steps)
            out[label]["loops"][kind] = c
            p = c["pipes"]
            print(f"  {kind:10s} loop ({steps} steps/iteration), per 4 steps: {c['instructions']:g} instructions | "
                  f"ALU {p['alu']:g} (= {c['alu_issue_cycles']:g} issue cycles at half rate)  FMA {p['fma']:g}  "
                  f"MIO {p['mio']:g}  other {p['other']:g}")
            ops = c["opcodes"] if args.opcodes else dict(list(c["opcodes"].items())[:12])
            for pi in ("alu", "fma", "mio", "other"):
                row = [f"{op} {n:g}" for op, n in ops.items() if pipe(op) == pi]
                if row:
                    print(f"    {pi:5s}: " + ", ".join(row))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
