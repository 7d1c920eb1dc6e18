#!/usr/bin/env python
"""Static SASS summary of the quadruped hot path in the step kernel (env_step_kernel_t<true>): for the RK4 step of the
quadruped signature, the composite-rigid-body evaluation, the one-call RK4 stage and the linear FSAL repair, print the
instruction count, the FP64 instruction count, basic blocks, local-memory traffic (STL / LDL), calls into the library's
division / square-root / trigonometric slow paths, and the spills ptxas reports.  The rows below them are the same
functions of the force-carrying hot path (env_step_kernel_ext: the RK4 and Euler steps, the evaluation and the stage with
the external-force slots applied).  The last rows are the same functions in the instances of batches with per-env model
rows (env_step_kernel_model_fast, env_step_kernel_model_ext).

Usage: python tools/hot_path_sass.py [--lib LIB.so [--ptxas-log LOG]]
Without --lib the library is compiled from the tree into a temporary directory (with -Xptxas -v, for the spills).
With --lib the spill column comes from --ptxas-log when given, else it is left out."""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL = "_ZN2jb17env_step_kernel_tILb1EEEvNS_10LaunchArgsE"
KERNEL_EXT = "_ZN2jb19env_step_kernel_extENS_10LaunchArgsE"
KERNEL_MODEL_FAST = "_ZN2jb26env_step_kernel_model_fastENS_10LaunchArgsE"
KERNEL_MODEL_EXT = "_ZN2jb25env_step_kernel_model_extENS_10LaunchArgsE"
FUNCS = [("step_rk4_t<FastOf<SigQuadruped>>", KERNEL, "_ZN2jb10step_rk4_tINS_6FastOfINS_13SigQuadrupedTILb0EEEEEEEvNS_3CtxEdPi"),
         ("rhs_quadruped_crba", KERNEL, "_ZN2jb18rhs_quadruped_crbaENS_3CtxEbPi"),
         ("stage_quadruped_crba", KERNEL, "_ZN2jb20stage_quadruped_crbaENS_3CtxEdiiiidPi"),
         ("repair_quadruped_crba", KERNEL, "_ZN2jb21repair_quadruped_crbaENS_3CtxE"),
         ("step_rk4_t<FastOf<SigQuadrupedExt>>", KERNEL_EXT, "_ZN2jb10step_rk4_tINS_6FastOfINS_15SigQuadrupedExtEEEEEvNS_3CtxEdPi"),
         ("step_euler_t<FastOf<SigQuadrupedExt>>", KERNEL_EXT, "_ZN2jb12step_euler_tINS_6FastOfINS_15SigQuadrupedExtEEEEEvNS_3CtxEdPi"),
         ("rhs_quadruped_crba_ext", KERNEL_EXT, "_ZN2jb22rhs_quadruped_crba_extENS_3CtxEbPi"),
         ("stage_quadruped_crba_ext", KERNEL_EXT, "_ZN2jb24stage_quadruped_crba_extENS_3CtxEdiiiidPi")]
FUNCS += [(name + " [model]", {KERNEL: KERNEL_MODEL_FAST, KERNEL_EXT: KERNEL_MODEL_EXT}[k], m) for name, k, m in FUNCS]
FP64 = {"DFMA", "DMUL", "DADD", "DSETP", "DMNMX"}


def build(tmp):
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    lib = os.path.join(tmp, "libjiminy_b200.so")
    srcs = [os.path.join(g.CSRC, f) for f in ("jb_capi.cu", "jb_plan.cpp")]
    r = subprocess.run([g._nvcc()] + g.NVCC_FLAGS + ["-Xptxas", "-v", "-o", lib] + srcs + ["-ccbin", "/usr/bin/g++"],
                       capture_output=True, text=True, check=True)
    return lib, r.stdout + r.stderr


def spills(log):
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            out[cur] = int(m.group(1)) + int(m.group(2))
            cur = None
    return out


def disassemble(lib, tmp):
    subprocess.run(["cuobjdump", "-xelf", "all", os.path.abspath(lib)], cwd=tmp, check=True, capture_output=True)
    cubin = max((os.path.join(tmp, f) for f in os.listdir(tmp) if f.endswith(".cubin")), key=os.path.getsize)
    return subprocess.run(["nvdisasm", "-c", cubin], capture_output=True, text=True, check=True).stdout.splitlines()


def body(lines, kernel, mangled):
    head = f"${kernel}${mangled}:"
    try:
        start = lines.index(head)
    except ValueError:
        return None
    end = next((i for i in range(start + 1, len(lines)) if re.match(r"^(\.text|\$\S+:$)", lines[i])), len(lines))
    return lines[start + 1:end]


def summary(fn):
    ins = [l for l in fn if re.match(r"^\s+/\*[0-9a-f]{4,}\*/", l)]
    op = [re.sub(r"^\s+/\*[0-9a-f]+\*/\s+(@!?U?P[T\d]\s+)?", "", l).split()[0].split(".")[0] for l in ins]
    cnt = collections.Counter(op)
    calls = collections.Counter(m.group(1) for l in ins for m in [re.search(r"CALL\S*\s+`\(\S*?(__internal[\w$]*)\)", l)] if m)
    return {"instructions": len(ins), "fp64": sum(cnt[o] for o in FP64),
            "basic_blocks": 1 + sum(1 for l in fn if re.match(r"^\.L_x_\d+:", l)),
            "STL": cnt["STL"], "LDL": cnt["LDL"],
            "slow_path_calls": sum(calls.values()),
            "trig_calls": sum(v for k, v in calls.items() if "trig" in k),
            "calls_by_target": dict(calls)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--lib")
    ap.add_argument("--ptxas-log")
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        if a.lib:
            lib, log = a.lib, (open(a.ptxas_log).read() if a.ptxas_log else None)
        else:
            lib, log = build(tmp)
        lines = disassemble(lib, tmp)
    sp = spills(log) if log is not None else {}
    print(f"library: {lib}")
    cols = ["instructions", "fp64", "basic_blocks", "STL", "LDL", "slow_path_calls", "trig_calls", "spill_bytes"]
    print(f"{'function':<38}" + "".join(f"{c:>16}" for c in cols))
    for name, kernel, mangled in FUNCS:
        fn = body(lines, kernel, mangled)
        if fn is None:
            print(f"{name:<38}  (not in this library)")
            continue
        s = summary(fn)
        s["spill_bytes"] = sp.get(mangled, "n/a")
        print(f"{name:<38}" + "".join(f"{s[c]:>16}" for c in cols) + f"   {s['calls_by_target']}")


if __name__ == "__main__":
    main()
