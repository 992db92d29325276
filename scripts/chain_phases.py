#!/usr/bin/env python3
"""Where a launch of the benchmark's chain kernel goes: per-warp phase clocks on the GPU, and
the per-phase instruction counts that need no GPU.

    python scripts/chain_phases.py [--lib SO] [--steps K] [--regions R]   # GPU: phase clocks
    python scripts/chain_phases.py --sass [--lib SO]                      # SASS per phase
    python scripts/chain_phases.py --paths [--batch B]                    # host build: path shares per warp

GPU mode compiles an instrumented copy of the library (__graft_entry__.compile_library with
-DPK_CHAIN_PHASE_CLOCKS) into a temporary directory, or takes the one given with --lib, and
loads it in place of pink_b200/libpink_b200.so.  It runs the bench.py workload (UR5, same seed,
B = 65536, 32 rotating input sets, PDL as the library launches it) as one CUDA graph of K
launches, R times, and reads back after each the records of all its launches: for every
warp the %globaltimer and clock64 values at kernel entry, once q and the targets row have landed
(before the first step), after ChainStep::assemble, after the corner test of BoxLSQChol::corner_start, after the closed-form releases, after the rounds, after
griddepcontrol.wait and after the last store (pk_math.cuh, ChainPhase).  A mark holds the largest
value over the warp's lanes, so a phase of a warp lasts until its slowest lane is through.  It
prints, per phase, the median and p99 duration per warp, the span from the first warp's entry
to the last warp's end, the share of warps in which at least one lane enters each stage, and
the CTAs that entered well before their launch's median CTA (--early-ns): how many per launch,
their blockIdx.x, their lead, how long they wait, and the load phase of those CTAs against the
rest of the launch.

--sass attributes every SASS instruction of ik_chain_kernel<6, 1, true, true> to a phase by the
outermost source line of its inlining chain (nvdisasm -gi on a -lineinfo build).  --paths runs
the host build of the kernel bodies with the PK_COUNT_ITERS hooks over the same workload and
counts, per warp of 32 consecutive instances, which QP stages at least one lane takes.

Nothing is written to the tree.
"""

import argparse
import ctypes as C
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from __graft_entry__ import compile_library  # noqa: E402

CSRC = os.path.join(ROOT, "pink_b200", "csrc")
PHASES = ["entry", "loaded", "assemble", "corner", "closed_form", "rounds", "wait", "store"]
FLAGS = {"release1": 1, "release2": 2, "rounds": 4}
KERNEL = "ik_chain_kernel<6, 1, true, true>"
MAX_WARPS = 65536  # pk::kChainPhaseMaxWarps


class Record(C.Structure):  # pk::ChainPhaseRecord
    _fields_ = [("ns", C.c_uint64 * len(PHASES)), ("clk", C.c_uint64 * len(PHASES)), ("smid", C.c_uint32),
                ("flags", C.c_uint32), ("cta", C.c_uint32), ("pad", C.c_uint32)]


def build_instrumented(out_dir):
    so = os.path.join(out_dir, "libpink_b200.so")
    compile_library(ROOT, so, ["-DPK_CHAIN_PHASE_CLOCKS"])
    return so


def gpu_phases(args):
    import torch

    so = args.lib or build_instrumented(tempfile.mkdtemp(prefix="pk_phases_"))
    from pink_b200 import _cabi

    _cabi._LIB_PATH = os.path.abspath(so)
    lib = _cabi.load()
    if not hasattr(lib, "pk_chain_phase_records"):
        raise RuntimeError(f"{so} was built without PK_CHAIN_PHASE_CLOCKS")
    lib.pk_chain_phase_records.restype = C.c_int
    lib.pk_chain_phase_records.argtypes = [C.c_void_p, C.c_int, C.c_int]

    from pink_b200 import BatchedIK, FrameTask, PostureTask, workloads
    from pink_b200.engine import get_engine
    from pink_b200.limits import ConfigurationLimit, VelocityLimit
    from pink_b200.robots import load_robot_description

    device = torch.device("cuda", 0)
    model = load_robot_description("ur5_description").model
    eng = get_engine(model, device)
    table = eng.table
    B, NBUF = args.batch, 32
    f = table.frame_names.index("tool0")
    rng = np.random.default_rng(workloads.SEED)  # bench.py, rank 0
    qs, ts, vs, ss = [], [], [], []
    for _ in range(NBUF):
        q = workloads.sample_configurations(table, B, rng)
        qt = workloads.perturb_configurations(table, q, rng)
        oMf, _ = eng.forward_kinematics(torch.as_tensor(qt, dtype=torch.float32, device=device))
        qs.append(torch.as_tensor(q, dtype=torch.float32, device=device))
        ts.append(oMf[:, f].reshape(B, 12).contiguous())
        vs.append(torch.empty((B, 6), dtype=torch.float32, device=device))
        ss.append(torch.empty((B,), dtype=torch.int32, device=device))
    frame_task = FrameTask("tool0", position_cost=1.0, orientation_cost=1.0, lm_damping=1.0)
    frame_task.set_target(ts[0])
    posture_task = PostureTask(cost=1e-3)
    posture_task.set_target(workloads.ur5_posture_reference(model))
    ik = BatchedIK(model, [frame_task, posture_task], workloads.UR5_DT, damping=workloads.UR5_DAMPING,
                   limits=[ConfigurationLimit(model), VelocityLimit(model)], safety_break=True, device=device,
                   batch_size=B)
    kname = ik.kernel_name() if hasattr(ik, "kernel_name") else KERNEL

    def step(k):
        i = k % NBUF
        ik.solve(qs[i], ts[i], vs[i], ss[i])

    for k in range(5):
        step(k)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream(device)
    side.wait_stream(torch.cuda.current_stream(device))
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            for k in range(args.steps):
                step(k)
    torch.cuda.current_stream(device).wait_stream(side)
    g.replay()
    torch.cuda.synchronize()

    nw = (B + 31) // 32
    if args.steps * nw > MAX_WARPS:
        raise SystemExit(f"--steps {args.steps}: at most {MAX_WARPS // nw} launches of {nw} warps fit the records")
    buf = (Record * MAX_WARPS)()
    dt = np.dtype([("ns", "<u8", len(PHASES)), ("clk", "<u8", len(PHASES)), ("smid", "<u4"), ("flags", "<u4"),
                   ("cta", "<u4"), ("pad", "<u4")])
    lib.pk_chain_phase_records(C.addressof(buf), MAX_WARPS, 4)  # drop the warm-up's records
    regions = []
    for _ in range(args.regions):
        g.replay()
        torch.cuda.synchronize()
        n = lib.pk_chain_phase_records(C.addressof(buf), MAX_WARPS, 4)  # 128 threads per CTA
        if n != args.steps * nw:
            raise RuntimeError(f"pk_chain_phase_records returned {n} records, expected {args.steps * nw}")
        # CTAs take slots in the order they start, and every CTA of a launch starts before the
        # next launch's first: row k is launch k of the graph
        regions.append(np.frombuffer(buf, dtype=dt, count=n).copy().reshape(args.steps, nw))
    bad = int(sum(int((s != 0).sum().item()) for s in ss))
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    report(regions, kname, B, args, gpu, bad)


def report(regions, kname, B, args, gpu, bad):
    # every launch but the first of each replay, which has no predecessor to overlap
    rec = np.concatenate([r[1:].reshape(-1) for r in regions])
    ns, clk, flags = rec["ns"].astype(np.int64), rec["clk"].astype(np.int64), rec["flags"]
    CF, RD = PHASES.index("closed_form"), PHASES.index("rounds")
    done = (ns > 0).all(axis=1)  # every warp passes every mark in this workload
    total_clk = clk[done, -1] - clk[done, 0]
    total_ns = ns[done, -1] - ns[done, 0]
    cyc_per_ns = float(np.median(total_clk / np.maximum(total_ns, 1)))
    print(f"# {kname}: per-warp phase clocks of launches 2..{args.steps} of a {args.steps}-launch CUDA graph, "
          f"{args.regions} graph replays, {regions[0].shape[1]} warps per launch (B = {B}, bench.py workload and seed, PDL)")
    print(f"# GPU (name, power limit, max SM clock): {gpu}")
    print(f"# warps with every mark: {int(done.sum())} of {len(rec)}; nonzero status over the inputs: {bad}")
    ns, clk, flags = ns[done], clk[done], flags[done]
    print(f"# durations per warp from clock64, converted at the measured {cyc_per_ns:.3f} cycles/ns")
    print(f"{'phase':<34}{'median ns':>10}{'p99 ns':>10}{'mean ns':>10}{'share of median warp':>22}")
    med_total = float(np.median(total_clk)) / cyc_per_ns
    for k in range(1, len(PHASES)):
        d = (clk[:, k] - clk[:, k - 1]) / cyc_per_ns
        print(f"{PHASES[k - 1] + ' -> ' + PHASES[k]:<34}{np.median(d):>10.0f}{np.quantile(d, 0.99):>10.0f}"
              f"{d.mean():>10.0f}{np.median(d) / med_total:>22.1%}")
    work = (clk[:, RD] - clk[:, 0]) / cyc_per_ns
    common = (clk[:, CF] - clk[:, 0]) / cyc_per_ns
    print(f"{'entry -> store (whole warp)':<34}{med_total:>10.0f}{np.quantile(total_clk, 0.99) / cyc_per_ns:>10.0f}"
          f"{total_clk.mean() / cyc_per_ns:>10.0f}")
    print(f"{'entry -> rounds (before the wait)':<34}{np.median(work):>10.0f}{np.quantile(work, 0.99):>10.0f}"
          f"{work.mean():>10.0f}")
    print(f"# entry -> closed_form (loads + assemble + corner + releases), median warp: {np.median(common):.0f} ns = "
          f"{np.median(common) / np.median(work):.1%} of the median entry -> rounds, "
          f"{np.median(common) / med_total:.1%} of the median entry -> store")
    only1 = (flags & 6) == 0
    if only1.any():
        c1 = (clk[only1, CF] - clk[only1, 0]) / cyc_per_ns
        w1 = (clk[only1, RD] - clk[only1, 0]) / cyc_per_ns
        print(f"# warps with no second release and no rounds ({only1.mean():.1%}): assemble + corner + first release "
              f"median {np.median(c1):.0f} ns of {np.median(w1):.0f} ns before the wait")
    spans, works, gaps = [], [], []
    for r in regions:
        n = r["ns"].astype(np.int64)
        for k in range(1, n.shape[0]):
            spans.append(n[k, :, -1].max() - n[k, :, 0].min())
            works.append(n[k, :, RD].max() - n[k, :, 0].min())
            gaps.append(n[k, :, -1].max() - n[k - 1, :, -1].max())
    print(f"# per launch (globaltimer): first warp entry -> last warp store median {np.median(spans):.0f} ns "
          f"(min {np.min(spans):.0f}, max {np.max(spans):.0f}); first entry -> last warp past the rounds median "
          f"{np.median(works):.0f} ns; last store of the previous launch -> last store median {np.median(gaps):.0f} ns")
    for name, bit in FLAGS.items():
        print(f"# warps with at least one lane in {name:<9}: {np.mean((flags & bit) != 0):.1%}")
    early_ctas(regions, cyc_per_ns, args.early_ns)


def early_ctas(regions, cyc_per_ns, lead_ns):
    """CTAs that entered at least `lead_ns` before their launch's median CTA entry: how many per
    launch, which blockIdx.x, how far ahead and how long their warps wait at griddepcontrol.wait;
    and the load phase of the early CTAs against the rest (the burst)."""
    LD, RD, WT = PHASES.index("loaded"), PHASES.index("rounds"), PHASES.index("wait")
    counts, lowest, blocks, leads, waits, ld_early, ld_burst = [], [], [], [], [], [], []
    for r in regions:
        for k in range(1, r.shape[0]):
            rec = r[k]
            cta = rec["cta"].astype(np.int64)
            ns, clk = rec["ns"].astype(np.int64), rec["clk"].astype(np.int64)
            n = int(cta.max()) + 1
            entry = np.full(n, np.iinfo(np.int64).max)
            np.minimum.at(entry, cta, ns[:, 0])
            lead = np.median(entry) - entry  # ns ahead of the median CTA entry
            early = np.flatnonzero(lead >= lead_ns)
            counts.append(len(early))
            lowest.append(len(early) == 0 or int(early.max()) == len(early) - 1)
            blocks.extend(early.tolist())
            leads.extend(lead[early].tolist())
            w_early = np.isin(cta, early)
            waits.extend(((clk[w_early, WT] - clk[w_early, RD]) / cyc_per_ns).tolist())
            ld = (clk[:, LD] - clk[:, 0]) / cyc_per_ns
            ld_early.extend(ld[w_early].tolist())
            ld_burst.extend(ld[~w_early].tolist())
    counts = np.array(counts)
    print(f"# early CTAs (entry >= {lead_ns / 1e3:g} us before the launch's median CTA entry): per launch median "
          f"{np.median(counts):.0f} (min {counts.min()}, max {counts.max()}) over {len(counts)} launches; "
          f"launches whose early CTAs are exactly blockIdx.x 0 .. count - 1: {np.mean(lowest):.1%}")
    if not blocks:
        return
    b = np.array(blocks)
    print(f"# early CTAs' blockIdx.x: min {b.min()}, median {np.median(b):.0f}, max {b.max()}; lead over the median "
          f"entry median {np.median(leads):.0f} ns (min {np.min(leads):.0f}, max {np.max(leads):.0f}); their warps' "
          f"rounds -> wait median {np.median(waits):.0f} ns (p99 {np.quantile(waits, 0.99):.0f})")
    print(f"# entry -> loaded, median warp: early CTAs {np.median(ld_early):.0f} ns (p99 "
          f"{np.quantile(ld_early, 0.99):.0f}), the other CTAs {np.median(ld_burst):.0f} ns (p99 "
          f"{np.quantile(ld_burst, 0.99):.0f})")


# ---- SASS per phase ---------------------------------------------------------------------------


def _ranges(csrc):
    """(file, first line, last line, phase) of the functions that define the phases."""
    def lines(name):
        return open(os.path.join(csrc, name)).read().splitlines()

    def find(ls, pat, start=0):
        for k in range(start, len(ls)):
            if re.search(pat, ls[k]):
                return k + 1
        raise RuntimeError(f"pattern {pat!r} not found")

    ch, lsq, cabi = lines("pk_chain.cuh"), lines("pk_lsq.cuh"), lines("pk_cabi.cu")
    a0 = find(ch, r"PK_HD int assemble\(")
    a1 = find(ch, r"^  return status;", a0)
    c0 = find(lsq, r"static PK_HD bool corner_start\(")
    c1 = find(lsq, r"if \(act == ALL && neg == 0u\) return false;", c0)
    f1 = find(lsq, r"// Gram matrix H = A\^T A", c1)
    g0 = find(lsq, r"static PK_HD void gram\(")
    g1 = find(lsq, r"// Whole solve in one thread", g0)
    k0 = find(cabi, r"ik_chain_kernel\(const __grid_constant__")
    k1 = find(cabi, r"^// Solve to a tolerance on chains", k0)
    return [("pk_chain.cuh", a0, a1, "assemble"), ("pk_lsq.cuh", c0, c1, "corner"),
            ("pk_lsq.cuh", c1 + 1, f1, "closed_form"), ("pk_lsq.cuh", g0, g1, "rounds"),
            ("pk_cabi.cu", k0, k1, "kernel: loads, PDL, stores")]


def sass_phases(args):
    so = args.lib or os.path.join(ROOT, "pink_b200", "libpink_b200.so")
    tmp = tempfile.mkdtemp(prefix="pk_sass_")
    subprocess.run(["cuobjdump", "-xelf", "all", os.path.abspath(so)], cwd=tmp, check=True, capture_output=True)
    cubins = [os.path.join(tmp, f) for f in os.listdir(tmp) if f.endswith(".cubin")]
    sym = None
    for cb in cubins:
        names = subprocess.run(["cuobjdump", "-symbols", cb], capture_output=True, text=True).stdout
        for m in re.finditer(r"(_ZN2pk\d+ik_chain_kernelILi6ELi1ELb1ELb1EE\S*)", names):
            sym, cubin = m.group(1), cb
    if sym is None:
        raise RuntimeError("ik_chain_kernel<6, 1, true, true> not found")
    full = subprocess.run(["nvdisasm", "-gi", cubin], capture_output=True, text=True, check=True).stdout
    start = full.index(f".section\t.text.{sym},")
    end = full.find(".section\t", start + 1)
    text = full[start:end if end > 0 else len(full)]
    ranges = _ranges(args.src or CSRC)
    # nvdisasm prints one "//## File" line per level of the inlining chain, innermost first
    counts, frames, fresh = {}, [], True
    loc = re.compile(r'//## File "([^"]+)", line (\d+)(?: inlined at "([^"]+)", line (\d+))?')
    for line in text.splitlines():
        m = loc.search(line)
        if m:
            if fresh:
                frames, fresh = [], False
            frames.append((os.path.basename(m.group(1)), int(m.group(2))))
            if m.group(3):
                frames.append((os.path.basename(m.group(3)), int(m.group(4))))
            continue
        if re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+\S", line) and ";" in line:
            fresh = True
            phase = "other"
            for f, n in reversed(frames):  # the outermost frame inside a phase range decides
                hit = [p for (rf, r0, r1, p) in ranges if rf == f and r0 <= n <= r1]
                if hit:
                    phase = hit[0]
                    if phase != "kernel: loads, PDL, stores":
                        break
            counts[phase] = counts.get(phase, 0) + 1
    total = sum(counts.values())
    print(f"# {KERNEL}: static SASS instructions per phase ({os.path.basename(so)}, nvdisasm -gi, outermost source frame)")
    for p in ["assemble", "corner", "closed_form", "rounds", "kernel: loads, PDL, stores", "other"]:
        print(f"{p:<30}{counts.get(p, 0):>7}")
    print(f"{'total':<30}{total:>7}")


# ---- path shares per warp (host build) -------------------------------------------------------


def host_paths(args):
    so = os.path.join(tempfile.mkdtemp(prefix="pk_paths_"), "pk_paths.so")
    src = os.path.join(tempfile.mkdtemp(prefix="pk_paths_src_"), "hooks.cpp")
    with open(src, "w") as fh:
        fh.write(PATH_HOOKS.replace("@HOSTSIM@", os.path.join(ROOT, "tests", "hostsim", "hostsim.cpp")))
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-ffp-contract=off",
                           "-I", os.path.join(ROOT, "tests", "hostsim"), "-o", so, src])
    import tests.hostsim as hsmod

    hsmod._lib = C.CDLL(so)
    hsmod._lib.hs_last_error.restype = C.c_char_p
    hsmod._lib.pk_path_tags.restype = C.c_int
    from tests import helpers
    from tests.hostsim import HostSim

    sc = helpers.ur5_scenario(args.batch, "reachable")
    hs = HostSim(sc.model)
    prob, targets, _ = sc.problem()
    hs.solve_ik(prob, sc.q32, targets, path=0)
    tags = np.zeros(args.batch, dtype=np.int32)
    n = hsmod._lib.pk_path_tags(tags.ctypes.data_as(C.c_void_p), args.batch)
    tags = tags[:n]
    # tag per instance: 0 optimal at the corner, 1 one release, 2 two releases, 3 rounds
    w = tags[: len(tags) // 32 * 32].reshape(-1, 32)
    print(f"# host build, UR5 benchmark workload ({n} instances, tests.helpers.ur5_scenario 'reachable'), "
          f"chain solver with the closed-form releases")
    for k, name in ((1, "first release"), (2, "second release"), (3, "rounds")):
        print(f"{name:<16} instances {np.mean(tags >= k):7.2%}   warps of 32 with at least one lane {np.mean((w >= k).any(axis=1)):7.2%}")


# The PK_COUNT_ITERS hooks of corner_start report, per instance, which closed-form exit it took
# (value 0 corner, 1 / 3 one release, 2 / 4 two releases, 11 / 12 / 14 rounds follow); the host
# solve runs the instances in order, so the n-th call belongs to instance n.
PATH_HOOKS = r"""
#include <vector>
static std::vector<int> g_tags;
extern "C" void pk_count_nfree(int v, int tag) {
  if (tag != -1 || v >= 100) return;
  g_tags.push_back(v == 0 ? 0 : (v == 1 || v == 3) ? 1 : (v == 2 || v == 4) ? 2 : 3);
}
extern "C" int pk_path_tags(int* out, int n) {
  int m = (int)g_tags.size() < n ? (int)g_tags.size() : n;
  for (int k = 0; k < m; ++k) out[k] = g_tags[k];
  g_tags.clear();
  return m;
}
#define PK_COUNT_ITERS 1
#include "@HOSTSIM@"
"""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", help="instrumented (GPU mode) or product (--sass) library; default: build / the tree's")
    ap.add_argument("--steps", type=int, default=20, help="launches per CUDA graph")
    ap.add_argument("--regions", type=int, default=20, help="graph replays; the last launch of each is recorded")
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--early-ns", type=float, default=2000.0,
                    help="a CTA entering at least this long before its launch's median CTA entry is early")
    ap.add_argument("--src", help="--sass: pink_b200/csrc the library was built from (default: the tree's)")
    ap.add_argument("--sass", action="store_true")
    ap.add_argument("--paths", action="store_true")
    args = ap.parse_args()
    if args.sass:
        sass_phases(args)
    elif args.paths:
        host_paths(args)
    else:
        gpu_phases(args)


if __name__ == "__main__":
    main()
