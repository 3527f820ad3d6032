#!/usr/bin/env python
"""step_sass_footprint.py -- how much SASS k_env_step<float, 16> runs per physics substep, per control step and per reset.  No GPU needed.

  python scripts/step_sass_footprint.py [--out FILE.json] [--csrc DIR] [--top 25]

Compiles step_kernel.cu for sm_90a with the flags of uhc_b200/build.py (-lineinfo, -Xptxas -v; UHC_NVCC_EXTRA is honoured) to a cubin in a
temporary directory, disassembles k_env_step<float, 16, false> and <float, 16, true> with `nvdisasm -gi`, and attributes every instruction:

  * to the subroutine it sits in: the kernel body or one of its out-of-line (__noinline__) functions, which the SASS names;
  * through the inline chain nvdisasm prints before it (innermost source line, then each call site it was inlined at) to the innermost
    function of the project's sources (CUDA's own headers are skipped).  Function extents come from the sources: every UHC_DEV / UHC_DEVNI /
    __device__ / __global__ definition, matched brace to brace.  Code the compiler merged across call sites carries one of their chains, so
    the split by function is close, not exact; the three sizes below do not depend on it except for the kernel body's own instructions.

Three static sizes per kernel (16 bytes per instruction):
  substep    the code a physics substep runs: substep_dynamics and every subroutine it calls (the PD, smooth and Newton phases, the solves,
             collide, the constraint set-up), and the kernel body's instructions inside env_step_warp's substep loop (the alignment barrier,
             integrate)
  step       the once-per-step set-up and epilogue: the rest of the kernel body (state load, action staging, body quaternions, reward,
             termination, observation, state store) and the subroutines only it calls (world_quat, called in the loop's last substep only,
             is counted here)
  reset      the in-kernel re-seed of finished episodes: the kernel body's instructions inlined from env_reset_warp and the subroutines
             only it calls (the reset's forward pass shares substep_dynamics with the substep and is counted there)

Writes the sizes, the subroutines, the largest innermost functions, the nvcc version and ptxas's registers and spills as JSON
(--out) and prints a table.
"""
import argparse
import collections
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
KERNELS = {"k_env_step<float,16,false>": "_Z10k_env_stepIfLi16ELb0EEvN3uhc10EngineViewIT_EEPKfPfS6_S6_PiS7_S6_S6_PKi",
           "k_env_step<float,16,true>": "_Z10k_env_stepIfLi16ELb1EEvN3uhc10EngineViewIT_EEPKfPfS6_S6_PiS7_S6_S6_PKi"}
SUBSTEP_ROOT = "substep_dynamics"
INS_BYTES = 16


def _blank(src):
    """the source with comments, string and character literals replaced by spaces (newlines kept, so offsets and lines still match)"""
    out, i, n = list(src), 0, len(src)
    while i < n:
        c = src[i]
        if src.startswith("//", i):
            j = src.find("\n", i)
            j = n if j < 0 else j
        elif src.startswith("/*", i):
            j = src.find("*/", i + 2)
            j = n if j < 0 else j + 2
        elif c in "\"'":
            j = i + 1
            while j < n and src[j] != c:
                j += 2 if src[j] == "\\" else 1
            j += 1
        else:
            i += 1
            continue
        for k in range(i, min(j, n)):
            if out[k] != "\n":
                out[k] = " "
        i = j
    return "".join(out)


NOT_NAMES = {"UHC_STEP_BOUNDS", "__launch_bounds__", "__maxnreg__", "alignas", "__align__", "sizeof", "decltype"}


def source_functions(path):
    """[(name, first line, last line)] of the device function definitions in one source file (1-based lines)"""
    s = _blank(open(path).read())
    line_of = lambda off: s.count("\n", 0, off) + 1
    res = []
    for m in re.finditer(r"\b(UHC_DEV|UHC_DEVNI|__global__|__device__)\b", s):
        ls = s.rfind("\n", 0, m.start()) + 1
        if s[ls:m.start()].lstrip().startswith("#"):
            continue                                          # a macro definition
        i, depth, name = m.end(), 0, None
        while i < len(s):
            c = s[i]
            if c == "(":
                if depth == 0:
                    j = i
                    while j > 0 and s[j - 1].isspace():
                        j -= 1
                    k = j
                    while k > 0 and (s[k - 1].isalnum() or s[k - 1] == "_"):
                        k -= 1
                    if s[k:j] and s[k:j] not in NOT_NAMES:
                        name = s[k:j]
                depth += 1
            elif c == ")":
                depth -= 1
            elif depth == 0 and c in ";{":
                break
            i += 1
        if i >= len(s) or s[i] != "{" or not name:
            continue                                          # a declaration
        d, j = 0, i
        while j < len(s):
            d += {"{": 1, "}": -1}.get(s[j], 0)
            if d == 0:
                break
            j += 1
        res.append((name, line_of(m.start()), line_of(j)))
    return res


class Sources:
    def __init__(self, csrc):
        self.csrc = os.path.realpath(csrc)
        self.funcs = {}

    def function(self, path, line):
        """the innermost function of the project's sources that holds path:line, or None (a CUDA header)"""
        rp = os.path.realpath(path)
        if os.path.dirname(rp) != self.csrc:
            return None
        if rp not in self.funcs:
            self.funcs[rp] = source_functions(rp) if os.path.exists(rp) else []
        best = None
        for name, a, b in self.funcs[rp]:
            if a <= line <= b and (best is None or b - a < best[2] - best[1]):
                best = (name, a, b)
        return best

    def loop_lines(self, fname, func, pattern):
        """the line range of the first `pattern` loop (a regex on its header line) inside function `func` of csrc/fname"""
        path = os.path.join(self.csrc, fname)
        s = _blank(open(path).read())
        lines = s.split("\n")
        f = [r for r in source_functions(path) if r[0] == func][0]
        for ln in range(f[1], f[2] + 1):
            if re.search(pattern, lines[ln - 1]):
                off = sum(len(x) + 1 for x in lines[:ln - 1])
                i = s.index("{", off)
                d, j = 0, i
                while True:
                    d += {"{": 1, "}": -1}.get(s[j], 0)
                    if d == 0:
                        break
                    j += 1
                return ln, s.count("\n", 0, j) + 1
        raise RuntimeError("no loop %r in %s" % (pattern, func))


CHAIN = re.compile(r'^\s*//## File "([^"]+)", line (\d+)(?: inlined at "([^"]+)", line (\d+))?')
INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")
CALL = re.compile(r"CALL\.(?:REL|ABS)(?:\.NOINC)?\s+`\(([^)]+)\)")


def parse_kernel(sass, mangled):
    """{subroutine: [(instruction text, chain)]} of one kernel's .text section; chain = [(file, line)] innermost first"""
    subs = collections.OrderedDict()
    cur, chain, pending, inside = None, [], [], False
    for l in sass.splitlines():
        if l.startswith(".text."):
            inside = l[6:].rstrip(":") == mangled
            if inside:
                cur = "<kernel body>"
                subs[cur] = []
            continue
        if not inside:
            continue
        if l.startswith(".section") or l.startswith("\t.section"):
            break
        m = re.match(r"^(\$[^:\s]+):\s*$", l)
        if m:
            cur = m.group(1)
            subs[cur] = []
            continue
        m = CHAIN.match(l)
        if m:
            pending.append((m.group(1), int(m.group(2))))
            continue
        m = INSN.match(l)
        if m:
            if pending:
                chain, pending = pending, []
            subs[cur].append((m.group(2), chain))
    return subs


def short_name(sub):
    if sub == "<kernel body>":
        return sub
    tail = sub.rsplit("$", 1)[-1]
    try:
        dm = subprocess.run(["c++filt", tail], capture_output=True, text=True).stdout.strip()
    except OSError:
        dm = tail
    dm = re.sub(r"^(?:void|int|bool|float|double)\s+", "", dm)
    return re.sub(r"\(.*$", "", dm).replace("uhc::", "")


def analyse(sass, mangled, srcs):
    subs = parse_kernel(sass, mangled)
    names = {s: short_name(s) for s in subs}
    calls = {s: set() for s in subs}
    for s, ins in subs.items():
        for text, _ in ins:
            m = CALL.search(text)
            if m and m.group(1) in subs:
                calls[s].add(m.group(1))
    loop = srcs.loop_lines("env_step.h", "env_step_warp", r"for \(int it = 0; it < NSUB")

    def reach(roots):
        seen, todo = set(), list(roots)
        while todo:
            s = todo.pop()
            if s not in seen:
                seen.add(s)
                todo.extend(calls[s])
        return seen

    # the kernel body's instructions: in the substep loop, in the reset, or the rest of the step
    body_part, body_calls = [], collections.defaultdict(set)
    for text, chain in subs["<kernel body>"]:
        fr = [srcs.function(f, ln) for f, ln in chain]
        part = "step"
        for (f, ln), fn in zip(chain, fr):
            if fn and fn[0] == "env_reset_warp":
                part = "reset"
                break
            if fn and fn[0] == "env_step_warp" and os.path.basename(f) == "env_step.h" and loop[0] <= ln <= loop[1]:
                part = "substep"
                break
        body_part.append(part)
        m = CALL.search(text)
        if m and m.group(1) in subs:
            body_calls[part].add(m.group(1))
    # substep_dynamics is the substep's code; the loop body's other call (world_quat, in the last substep only) runs once per step
    root = [s for s in subs if names[s].split("<")[0] == SUBSTEP_ROOT]
    substep_subs = reach(root)
    body_calls["step"] |= body_calls["substep"] - set(root)
    step_subs = reach(body_calls["step"]) - substep_subs
    reset_subs = reach(body_calls["reset"]) - substep_subs - step_subs
    part_of = {s: "substep" if s in substep_subs else "step" if s in step_subs else "reset" if s in reset_subs else "step" for s in subs}

    sizes = collections.Counter()
    by_sub, by_fn = collections.Counter(), collections.Counter()
    for s, ins in subs.items():
        for i, (text, chain) in enumerate(ins):
            part = body_part[i] if s == "<kernel body>" else part_of[s]
            sizes[part] += 1
            by_sub[(part, names[s])] += 1
            inner = next((fn[0] for fn in (srcs.function(f, ln) for f, ln in chain) if fn), "(CUDA runtime)")
            by_fn[(part, inner)] += 1
    kb = lambda n: round(n * INS_BYTES / 1024, 1)
    return dict(
        instructions=sum(sizes.values()), kbytes=kb(sum(sizes.values())),
        substep_kbytes=kb(sizes["substep"]), step_kbytes=kb(sizes["step"]), reset_kbytes=kb(sizes["reset"]),
        instructions_by_part=dict(sizes),
        subroutines=[dict(part=p, name=n, instructions=c, kbytes=kb(c)) for (p, n), c in by_sub.most_common()],
        functions=[dict(part=p, function=f, instructions=c, kbytes=kb(c)) for (p, f), c in by_fn.most_common()],
        substep_loop_lines=list(loop))


def ptxas_info(text):
    """{mangled function: dict(stack, spill_stores, spill_loads[, registers for an entry])} from nvcc -Xptxas -v output"""
    res, cur, props = {}, None, None
    for l in text.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", l)
        if m:
            cur = m.group(1)
            res[cur] = {}
            continue
        m = re.search(r"Function properties for (\S+)", l)
        if m:
            props = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", l)
        if m and props:
            res.setdefault(props, {}).update(stack=int(m.group(1)), spill_stores=int(m.group(2)), spill_loads=int(m.group(3)))
            continue
        m = re.search(r"Used (\d+) registers", l)
        if m and cur in res:
            res[cur]["registers"] = int(m.group(1))
    return res


def compile_cubin(csrc, tmp, defines=()):
    from uhc_b200 import build
    flags = [f for f in build.NVCC_FLAGS if f not in ("-shared", "--use_fast_math=false")]
    flags = [f for i, f in enumerate(flags) if not (f == "-Xcompiler" or (i and flags[i - 1] == "-Xcompiler"))]
    flags += os.environ.get("UHC_NVCC_EXTRA", "").split() + ["-D" + d for d in defines]
    cubin = os.path.join(tmp, "step_kernel.cubin")
    r = subprocess.run(["nvcc"] + flags + ["-cubin", "-o", cubin, os.path.join(csrc, "step_kernel.cu")], capture_output=True, text=True)
    if r.returncode:
        sys.stderr.write(r.stderr[-8000:])
        raise RuntimeError("nvcc failed")
    return cubin, r.stdout + r.stderr, flags


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="JSON file to write")
    ap.add_argument("--csrc", default=os.path.join(ROOT, "uhc_b200", "csrc"), help="source directory holding step_kernel.cu")
    ap.add_argument("--top", type=int, default=25, help="how many innermost functions to list")
    ap.add_argument("-D", dest="defines", action="append", default=[], help="extra preprocessor macro (NAME or NAME=VALUE)")
    a = ap.parse_args()
    srcs = Sources(a.csrc)
    with tempfile.TemporaryDirectory() as tmp:
        cubin, ptx_log, flags = compile_cubin(a.csrc, tmp, a.defines)
        sass = subprocess.run(["nvdisasm", "-gi", cubin], capture_output=True, text=True, check=True).stdout
    regs = ptxas_info(ptx_log)
    ver = subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-2:]
    res = dict(nvcc=" ".join(ver), flags=flags, bytes_per_instruction=INS_BYTES, kernels={})
    for label, mangled in KERNELS.items():
        r = analyse(sass, mangled, srcs)
        r["ptxas"] = regs.get(mangled, {})
        # out-of-line functions are compiled once per module and shared by every kernel that calls them
        subs = {sub.rsplit("$", 1)[-1] for sub in parse_kernel(sass, mangled)}
        r["ptxas_subroutines"] = {short_name("$" + k): v for k, v in regs.items() if k != mangled and k in subs}
        r["functions"] = r["functions"][:a.top]
        res["kernels"][label] = r
        print("%s: %d instructions (%.1f KB): substep %.1f KB, step set-up / epilogue %.1f KB, reset %.1f KB; ptxas %s" % (
            label, r["instructions"], r["kbytes"], r["substep_kbytes"], r["step_kbytes"], r["reset_kbytes"], r["ptxas"]))
        for s in r["subroutines"]:
            print("   %-8s %-28s %6d  %6.1f KB" % (s["part"], s["name"][:28], s["instructions"], s["kbytes"]))
        print("   largest innermost functions:")
        for f in r["functions"]:
            print("   %-8s %-49s %6d  %6.1f KB" % (f["part"], f["function"][:49], f["instructions"], f["kbytes"]))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
