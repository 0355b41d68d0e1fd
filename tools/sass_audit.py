"""Memory-space audit of the product library's SASS (CPU only: nvcc cross-compiles for sm_90a, no GPU needed).

Compiles smplsim_b200/csrc/smplsim_capi.cu to a cubin with the library's own nvcc flags, disassembles it with `nvdisasm -g`
and prints, per kernel instance: registers, stack frame, spill bytes (the entry plus the device functions ptxas reports after
it) and the counts of local (LDL / STL), generic (LD / ST), global (LDG / STG) and shared (LDS / STS) memory instructions.
Then, for the instances selected with --lines, the LDL sites by source line of lane_kernels.cuh (a stack load in front of a
global access is a second dependent round trip).

    python tools/sass_audit.py                      # table of all step / reset / kin / inverse / dyn instances
    python tools/sass_audit.py --lines "k_step5<24," ",0,0>"    # + LDL sites of the cfg2 step kernel (SMPL, no self-collision, no xfrc)
"""
from __future__ import annotations

import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from smplsim_b200 import _lib  # noqa: E402

CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
OPS = ("LDL", "STL", "LD", "ST", "LDG", "STG", "LDS", "STS")
KERNELS = ("k_step5", "k_reset5", "k_kin5", "k_inverse5", "k_dyn5")


def compile_cubin(out_dir: str) -> tuple[str, str]:
    """cubin path and the ptxas -v log."""
    flags = [f for f in _lib.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC")]
    cubin = os.path.join(out_dir, "lib.cubin")
    r = subprocess.run([os.path.join(CUDA, "bin", "nvcc")] + flags + ["-Xptxas", "-v", "-cubin", "-o", cubin, "smplsim_capi.cu"],
                       cwd=_lib._CSRC, capture_output=True, text=True, check=True)
    return cubin, r.stderr


def ptxas_stats(log: str) -> dict:
    """entry -> [registers, stack frame, spill stores, spill loads]; spills of the device functions listed after an entry are added to it."""
    stats, cur, fn = {}, None, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            stats[cur] = [0, 0, 0, 0]
            continue
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            if fn == cur:
                stats[cur][1] = int(m.group(1))
            stats[cur][2] += int(m.group(2))
            stats[cur][3] += int(m.group(3))
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m and cur:
            stats[cur][0] = int(m.group(1))
    return stats


def sass_counts(sass: str) -> tuple[dict, dict]:
    """entry -> Counter of memory opcodes; entry -> Counter of LDL sites by lane_kernels.cuh line."""
    counts, ldl = {}, {}
    cur, line_no = None, None
    for line in sass.splitlines():
        m = re.match(r"\s*\.section\s+\.text\.(\S+?),", line)
        if m:
            cur = m.group(1)
            counts[cur], ldl[cur] = collections.Counter(), collections.Counter()
            continue
        m = re.search(r'//## File "([^"]+)", line (\d+)', line)
        if m:
            line_no = int(m.group(2)) if m.group(1).endswith("lane_kernels.cuh") else None
            continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9]+)(\.[A-Z0-9.]+)?\s", line)
        if not m or cur is None:
            continue
        op = m.group(1)
        if op in OPS:
            counts[cur][op] += 1
            if op == "LDL":
                ldl[cur][line_no] += 1
    return counts, ldl


def short(name: str) -> str:
    m = re.match(r"_Z\d+(k_\w+?)I4LCfgI((?:Li\d+E)+)", name)
    if not m:
        return name
    return f"{m.group(1)}<{','.join(re.findall(r'Li(\d+)E', m.group(2)))}>"


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--lines", nargs="*", default=[], metavar="SUBSTR",
                    help="print LDL sites by source line for instances whose short name contains every SUBSTR")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as d:
        cubin, log = compile_cubin(d)
        sass = subprocess.run([os.path.join(CUDA, "bin", "nvdisasm"), "-g", "-c", cubin], capture_output=True, text=True, check=True).stdout
    stats = ptxas_stats(log)
    counts, ldl = sass_counts(sass)
    rows = sorted((short(n), n) for n in stats if any(k in n for k in KERNELS))
    print(f"{'instance':<48}{'regs':>5}{'stack':>6}{'spSt':>5}{'spLd':>5}" + "".join(f"{o:>6}" for o in OPS))
    for s, n in rows:
        r, st, ss, sl = stats[n]
        c = counts.get(n, collections.Counter())
        print(f"{s:<48}{r:>5}{st:>6}{ss:>5}{sl:>5}" + "".join(f"{c[o]:>6}" for o in OPS))
    if args.lines:
        for s, n in rows:
            if all(k in s for k in args.lines):
                print(f"\nLDL sites of {s} by lane_kernels.cuh line:")
                for ln, k in sorted(ldl[n].items(), key=lambda t: (t[0] is None, t[0] or 0)):
                    print(f"  line {ln if ln is not None else '?':>5}: {k}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
