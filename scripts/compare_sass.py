"""Compare the machine code of two builds of the CUDA library, kernel by kernel.

    python scripts/compare_sass.py [BASE_REV] [--out DIR]

Builds pink_b200/csrc/pk_cabi.cu of git revision BASE_REV (default HEAD) and of the working
tree with __graft_entry__.NVCC_FLAGS plus -Xptxas -v, in parallel, then compares for every
kernel:
  - the cuobjdump -sass listing, with the /*addr*/ comments stripped and whitespace collapsed;
  - ptxas' registers / barriers / shared and constant memory line and its stack frame / spill
    line.
A refactor of the host code must leave every kernel identical.  Kernels are matched by their
demangled name with the parameter list removed, so a kernel that gained a parameter is compared
with its old self ("signature changed").  Prints one line per kernel that differs, was added or
was removed, with the ptxas lines and SASS instruction counts of both builds for the kernels
that differ, then a summary; exits 1 on any difference.  Nothing is written to the tree: the
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
            # whitespace collapsed: cuobjdump pads its columns to the widest line of the whole listing
            kernels[name].append(" ".join(ADDR.sub("", line).split()))
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


def demangle(names):
    out = subprocess.run(["cu++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return dict(zip(names, out))


def strip_params(demangled):
    """`void f<6, 1, true>(A, B)` -> `f<6, 1, true>`: drop the trailing parameter list and the
    return type."""
    s = demangled.strip()
    if s.endswith(")"):
        depth = 0
        for k in range(len(s) - 1, -1, -1):
            depth += {")": 1, "(": -1}.get(s[k], 0)
            if depth == 0:
                s = s[:k]
                break
    return s[5:] if s.startswith("void ") else s


def n_instructions(lines):
    return sum(1 for line in lines if ";" in line and not line.startswith(("/*", ".")))


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
    # kernel key (name and template arguments) -> mangled name, per build
    keyed = {}
    for tag in ("base", "tree"):
        dm = demangle(sorted(sass[tag]))
        keyed[tag] = {strip_params(d): (m, d) for m, d in dm.items()}
    keys = sorted(set(keyed["base"]) | set(keyed["tree"]))
    differ = added = removed = 0
    for key in keys:
        if key not in keyed["base"]:
            added += 1
            print(f"ADDED: {key}")
            continue
        if key not in keyed["tree"]:
            removed += 1
            print(f"REMOVED: {key}")
            continue
        (mb, db), (mt, dt) = keyed["base"][key], keyed["tree"][key]
        problems = []
        if sass["base"][mb] != sass["tree"][mt]:
            problems.append("sass")
        if ptxas["base"].get(mb) != ptxas["tree"].get(mt):
            problems.append("ptxas")
        sig = " (signature changed)" if db != dt else ""
        if problems:
            differ += 1
            print(f"DIFFERS ({', '.join(problems)}){sig}: {key}")
            for tag, m in (("base", mb), ("tree", mt)):
                print(f"    {tag}: {n_instructions(sass[tag][m])} instructions; " + " | ".join(ptxas[tag].get(m, [])))
        elif sig:
            print(f"IDENTICAL{sig}: {key}")
    counts = defaultdict(int)
    for key in keyed["tree"]:
        counts[re.match(r"(?:\w+::)*(\w+)", key).group(1)] += 1
    print("kernels:", len(keyed["tree"]), dict(sorted(counts.items())))
    same = len(keys) - differ - added - removed
    print(f"{same} identical, {differ} differ, {added} added, {removed} removed (builds in {out})")
    sys.exit(1 if differ or added or removed else 0)


if __name__ == "__main__":
    main()
