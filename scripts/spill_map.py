"""Local-memory traffic of the step kernel's substep loop, from the compiler's output alone (no GPU needed).

Compiles csrc/b2q_api.cu for sm_90a with the library's flags plus -cubin -Xptxas -v (flags include -lineinfo), disassembles the cubin with
source lines and their inlining chains, and for each step-kernel instantiation prints ptxas's registers, stack and spill bytes.  For the chosen instantiation
(default: b2q_step_kernel<float, 0>, the one bench.py times) it then finds two loops by their backward branches:

  - the PGS sweep loop: the loop whose instructions come from the sweep's source lines in b2q_sim.cuh;
  - the substep loop: the innermost loop that contains the sweep loop.

and lists every LDL / STL in the substep loop's body with its address and source line, plus the instruction counts of both bodies.
Each pass through the substep loop executes its body once (the sweep loop's body runs once per sweep).  LDL / STL outside the
substep loop run once per control step and are counted separately.

  python scripts/spill_map.py [--src DIR] [--type float|double] [--feat 0|1] [--json PATH]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")
LINE = re.compile(r'^\s*//## File "([^"]+)", line (\d+)')   # with -gi: `... inlined at "<file>", line <n>` may follow
LABEL = re.compile(r"^(\.L_x_\d+):")
BRA = re.compile(r"\bBRA\b.*`\((\.L_x_\d+)\)")
FUNC = re.compile(r"^\.text\.(\S+):")
PTXAS_FN = re.compile(r"(?:Compiling entry function '|Function properties for )(\S+?)'?$")
PTXAS_SPILL = re.compile(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads")
PTXAS_REGS = re.compile(r"Used (\d+) registers")
STEP = re.compile(r"b2q_step_kernelI([fd])Li(\d)E")


def compile_cubin(src, out_dir):
    from paddlerobotics_b200 import build as b
    flags = [f for f in b.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC")]
    cubin = os.path.join(out_dir, "b2q_api.cubin")
    cmd = [os.path.join(CUDA, "bin", "nvcc")] + flags + ["-cubin", "-Xptxas", "-v", "-o", cubin, os.path.join(src, "b2q_api.cu")]
    log = subprocess.run(cmd, capture_output=True, text=True)
    if log.returncode != 0:
        sys.stderr.write(log.stderr)
        raise SystemExit("nvcc failed")
    stats, fn = {}, None
    for ln in log.stderr.splitlines():
        m = PTXAS_FN.search(ln)
        if m:
            fn = m.group(1)
            continue
        m = PTXAS_SPILL.search(ln)
        if m and fn:
            stats.setdefault(fn, {}).update(stack=int(m.group(1)), spill_stores=int(m.group(2)), spill_loads=int(m.group(3)))
        m = PTXAS_REGS.search(ln)
        if m and fn:
            stats.setdefault(fn, {})["registers"] = int(m.group(1))
    sass = subprocess.run([os.path.join(CUDA, "bin", "nvdisasm"), "-gi", "-c", cubin], capture_output=True, text=True, check=True).stdout
    return stats, sass


def parse_functions(sass):
    """{mangled name: (instructions [(addr, text, file, line, sim line)], labels {label: index of the next instruction})}

    file:line is the innermost source location; sim line is the first location of the inlining chain in b2q_sim.cuh (0 if none), so
    that an m_fma of b2q_math.cuh inlined into the sweep counts as a line of the sweep."""
    funcs, cur, chain, fresh = {}, None, [], True
    for ln in sass.splitlines():
        m = FUNC.match(ln)
        if m:
            cur = funcs.setdefault(m.group(1), ([], {}))
            continue
        if cur is None:
            continue
        m = LINE.match(ln)
        if m:
            if fresh:
                chain, fresh = [], False
            chain.append((m.group(1), int(m.group(2))))
            continue
        m = LABEL.match(ln)
        if m:
            cur[1][m.group(1)] = len(cur[0])
            continue
        m = INSN.match(ln)
        if m:
            f, line = chain[0] if chain else (None, 0)
            sim = next((l for fn, l in chain if fn.endswith("b2q_sim.cuh")), 0)
            cur[0].append((int(m.group(1), 16), m.group(2), f, line, sim))
            fresh = True
    return funcs


def loops(insns, labels):
    """[(first, last)] instruction-index ranges of the loops: a branch back to a label at or before it"""
    out = []
    for i, (_, text, _, _, _) in enumerate(insns):
        m = BRA.search(text)
        if m and m.group(1) in labels and labels[m.group(1)] <= i:
            out.append((labels[m.group(1)], i))
    return out


def sweep_lines(src):
    """source lines of the PGS sweep loop in substep(): from its `for (int it ...` up to its early-exit test"""
    lines = open(os.path.join(src, "b2q_sim.cuh")).read().splitlines()
    start = next(i for i, l in enumerate(lines) if "projected Gauss-Seidel, Bullet row order" in l)
    first = next(i for i in range(start, len(lines)) if "for (int it = 0; it < cf.iters; it++)" in lines[i])
    last = next(i for i in range(first, len(lines)) if "if (moved == T(0)) break;" in lines[i])
    return first + 1, last + 1


def is_local(text):
    op = text.split()[1] if text.startswith("@") else text.split()[0]
    return op.split(".")[0] in ("LDL", "STL"), op.split(".")[0]


def analyse(insns, labels, src):
    lo, hi = sweep_lines(src)
    in_sweep = lambda i: lo <= insns[i][4] <= hi
    cand = [(a, b) for a, b in loops(insns, labels) if sum(in_sweep(i) for i in range(a, b + 1)) * 2 > b - a + 1]
    if not cand:
        raise SystemExit("sweep loop not found")
    sweep = min(cand, key=lambda r: r[1] - r[0])
    outer = [(a, b) for a, b in loops(insns, labels) if a <= sweep[0] and b >= sweep[1] and (a, b) != sweep]
    if not outer:
        raise SystemExit("substep loop not found")
    sub = min(outer, key=lambda r: r[1] - r[0])
    local_in, local_out = [], {"LDL": 0, "STL": 0}
    for i, (addr, text, f, line, sim) in enumerate(insns):
        loc, op = is_local(text)
        if not loc:
            continue
        if sub[0] <= i <= sub[1]:
            local_in.append({"addr": "%05x" % addr, "kind": op, "op": text, "file": os.path.basename(f or "?"), "line": line, "sim_line": sim, "in_sweep": sweep[0] <= i <= sweep[1]})
        else:
            local_out[op] += 1
    return {
        "substep_loop_instructions": sub[1] - sub[0] + 1,
        "sweep_loop_instructions": sweep[1] - sweep[0] + 1,
        "ldl_per_substep": sum(1 for x in local_in if x["kind"] == "LDL"),
        "stl_per_substep": sum(1 for x in local_in if x["kind"] == "STL"),
        "ldl_outside_substep_loop": local_out["LDL"],
        "stl_outside_substep_loop": local_out["STL"],
        "local_in_substep_loop": local_in,
        "sweep_source_lines": [lo, hi],
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--src", default=os.path.join(ROOT, "paddlerobotics_b200", "csrc"), help="CUDA sources to compile")
    ap.add_argument("--type", choices=["float", "double"], default="float")
    ap.add_argument("--feat", type=int, choices=[0, 1], default=0)
    ap.add_argument("--json", default=None, help="also write the result as JSON to this path")
    args = ap.parse_args()
    src = os.path.abspath(args.src)
    with tempfile.TemporaryDirectory() as tmp:
        stats, sass = compile_cubin(src, tmp)
    funcs = parse_functions(sass)
    res = {"src": src, "kernels": {}}
    print("%-28s %9s %9s %12s %12s" % ("step kernel", "registers", "stack B", "spill st B", "spill ld B"))
    for name, st in sorted(stats.items()):
        m = STEP.search(name)
        if not m:
            continue
        key = "b2q_step_kernel<%s, %s>" % ({"f": "float", "d": "double"}[m.group(1)], m.group(2))
        res["kernels"][key] = st
        print("%-28s %9d %9d %12d %12d" % (key, st["registers"], st["stack"], st["spill_stores"], st["spill_loads"]))
    want = "b2q_step_kernelI%sLi%dE" % (args.type[0], args.feat)
    name = next(n for n in funcs if want in n)
    insns, labels = funcs[name]
    a = analyse(insns, labels, src)
    a["kernel"] = "b2q_step_kernel<%s, %d>" % (args.type, args.feat)
    a["instructions"] = len(insns)
    res["map"] = a
    print("\n%s: %d instructions; substep loop body %d, PGS sweep loop body %d (sweep = b2q_sim.cuh:%d-%d)" %
          (a["kernel"], len(insns), a["substep_loop_instructions"], a["sweep_loop_instructions"], *a["sweep_source_lines"]))
    print("per substep: %d LDL + %d STL in the loop body; once per control step outside it: %d LDL + %d STL" %
          (a["ldl_per_substep"], a["stl_per_substep"], a["ldl_outside_substep_loop"], a["stl_outside_substep_loop"]))
    for x in a["local_in_substep_loop"]:
        where = "%s:%d" % (x["file"], x["line"]) + ("" if x["file"] == "b2q_sim.cuh" or not x["sim_line"] else " (b2q_sim.cuh:%d)" % x["sim_line"])
        print("  %s  %-40s %s%s" % (x["addr"], x["op"], where, "  (in the sweep)" if x["in_sweep"] else ""))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
