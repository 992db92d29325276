"""Compare the machine code of two builds of the CUDA library, kernel by kernel.

    python scripts/compare_sass.py [BASE_REV] [--out DIR]

Builds pink_b200/csrc/pk_cabi.cu of git revision BASE_REV (default HEAD) and of the working
tree with __graft_entry__.NVCC_FLAGS plus -Xptxas -v, in parallel, then compares for every
kernel:
  - the cuobjdump -sass listing, with the /*addr*/ comments stripped;
  - ptxas' registers / barriers / shared and constant memory line and its stack frame / spill
    line.
A refactor of the host code must leave every kernel identical.  Prints one line per kernel
that differs and a summary; exits 1 on any difference.  Nothing is written to the tree: the
builds go to a temporary directory (or DIR).
"""

import argparse
import os
import re
import subprocess
import sys
import tempfile
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from __graft_entry__ import NVCC_FLAGS  # noqa: E402

ADDR = re.compile(r"/\*[0-9a-f]{4,}\*/")


def start_build(src_root, out_dir):
    so = os.path.join(out_dir, "libpink_b200.so")
    log = open(os.path.join(out_dir, "ptxas.txt"), "w")
    cmd = ["nvcc", *NVCC_FLAGS, "-Xptxas", "-v", "-o", so, os.path.join(src_root, "pink_b200", "csrc", "pk_cabi.cu")]
    return so, subprocess.Popen(cmd, cwd=src_root, stdout=log, stderr=subprocess.STDOUT)


def sass_by_kernel(so):
    text = subprocess.run(["cuobjdump", "-sass", so], check=True, capture_output=True, text=True).stdout
    kernels, name = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            kernels[name] = []
        elif name is not None:
            kernels[name].append(ADDR.sub("", line).rstrip())
    return kernels


def ptxas_by_kernel(log):
    info, name = defaultdict(list), None
    for line in open(log):
        m = re.search(r"Compiling entry function '(\S+)'|Function properties for (\S+)", line)
        if m:
            name = m.group(1) or m.group(2)
        elif name and ("stack frame" in line or "Used " in line):
            info[name].append(line.strip())
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("base", nargs="?", default="HEAD")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    out = args.out or tempfile.mkdtemp(prefix="pk_sass_")
    base_src = os.path.join(out, "base_src")
    os.makedirs(base_src, exist_ok=True)
    archive = subprocess.run(["git", "-C", ROOT, "archive", args.base, "pink_b200/csrc", "include"], check=True,
                             capture_output=True).stdout
    subprocess.run(["tar", "-x", "-C", base_src], input=archive, check=True)
    builds = {}
    for tag, src in (("base", base_src), ("tree", ROOT)):
        d = os.path.join(out, tag)
        os.makedirs(d, exist_ok=True)
        builds[tag] = (d,) + start_build(src, d)
    for tag, (d, so, proc) in builds.items():
        if proc.wait():
            sys.exit(f"{tag} build failed, see {d}/ptxas.txt")
    sass = {tag: sass_by_kernel(so) for tag, (_, so, _) in builds.items()}
    ptxas = {tag: ptxas_by_kernel(os.path.join(d, "ptxas.txt")) for tag, (d, _, _) in builds.items()}
    names = sorted(set(sass["base"]) | set(sass["tree"]))
    differ = 0
    for n in names:
        problems = []
        if sass["base"].get(n) != sass["tree"].get(n):
            problems.append("sass")
        if ptxas["base"].get(n) != ptxas["tree"].get(n):
            problems.append("ptxas")
        if problems:
            differ += 1
            print(f"DIFFERS ({', '.join(problems)}): {n}")
    counts = defaultdict(int)
    demangled = subprocess.run(["cu++filt"], input="\n".join(names), capture_output=True, text=True).stdout
    for line in demangled.splitlines():
        counts[re.search(r"(\w+)[<(]", line).group(1)] += 1
    print("kernels:", len(names), dict(sorted(counts.items())))
    print(f"{len(names) - differ} identical, {differ} differ (builds in {out})")
    sys.exit(1 if differ else 0)


if __name__ == "__main__":
    main()
