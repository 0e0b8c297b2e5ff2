#!/usr/bin/env python
"""Where the time of the staged block kernel goes: a device-side clock at its phase boundaries, on the GPU.

Compiles an instrumented copy of the engine (build()'s nvcc flags plus -DB200PF_PHASE_CLOCK, csrc/b200pf_block.cuh) into
--out, loads it through B200PF_LIB and runs the bench.py workload: l2rpn_case14_sandbox AC, batch 4096, DoNothing on the
series path, L2 flushed between steps, --warmup steps, then --steps timed ones.  Lane 0 of every warp adds the SM cycles
between consecutive phase boundaries of solve_block to device counters; after every step they are read and cleared.  A
phase's time in a step is its cycle sum over the warps / the number of warps, converted to microseconds with the clock rate
the same warps measured (their globaltimer span over their clock64 span).  Prints one JSON line with the median over the steps.

    python scripts/phase_clock.py [--out DIR] [--lib PREBUILT.so] [--steps 200] [--warmup 10] [--batch 4096]

The instrumented kernel reads the clock 3 + 3 x iterations times per warp, so its phases add up to a little more than the
production kernel's step; use the table for where the time goes, bench.py for how long a step takes."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
GOLD = os.path.join(REPO, "tests", "golden")

# counters of b200pf_block.cuh (PC_*), in order
PHASES = ["stage", "row", "sums", "dc_inverse", "dc_angles", "nr_buses_vote", "nr_stream", "nr_update", "outputs"]
WHAT = {"stage": "kernel entry -> plan + static arrays staged (staged launches: the first rows are loaded meanwhile)",
        "row": "chronics row into the workspace (when not loaded during the staging)",
        "sums": "phase 1: per-bus sums of the injections, DC right-hand side",
        "dc_inverse": "DC angles = plan inverse x right-hand side",
        "dc_angles": "angles into the workspace, sincos, clearing of the fill-in blocks",
        "nr_buses_vote": "Newton, all iterations: I = Y V from the admittance rows, S(V), mismatch, the bus's block row "
                         "(diagonal + off-diagonal blocks), convergence vote (lane = bus)",
        "nr_stream": "Newton, all iterations: block LU + solves (the plan's operation stream)",
        "nr_update": "Newton, all iterations: state update, clearing of the fill-in blocks (lane = bus)",
        "outputs": "loop exit -> branch currents, result records, rho stored"}
N_SLOTS = len(PHASES) + 4          # + solves, warps, cycles, ns


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def build_instrumented(out_dir):
    from __graft_entry__ import NVCC_FLAGS
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        nvcc = "nvcc"
    lib = os.path.join(out_dir, "libb200pf_phase_clock.so")
    src = os.path.join(REPO, "grid2op_b200", "csrc", "b200pf.cu")
    subprocess.check_call([nvcc] + NVCC_FLAGS + ["-DB200PF_PHASE_CLOCK", "-o", lib, src])
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory of the instrumented library (default: a new temporary directory)")
    ap.add_argument("--lib", default=None, help="an instrumented library built before (skips the compile)")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--batch", type=int, default=4096)
    args = ap.parse_args()
    lib_file = args.lib
    if lib_file is None:
        out = args.out or tempfile.mkdtemp(prefix="b200pf_phase_clock_")
        os.makedirs(out, exist_ok=True)
        lib_file = build_instrumented(out)
    os.environ["B200PF_LIB"] = os.path.abspath(lib_file)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("phase_clock.py: no CUDA device (this measurement has no CPU fallback)")
    from grid2op_b200 import engine
    from grid2op_b200.gridmodel import GridModel
    from grid2op_b200.rollout import BatchedDoNothing
    lib = engine.load_library()
    if not hasattr(lib, "b200pf_phase_clock_read"):
        raise SystemExit(f"phase_clock.py: {lib_file} was not built with -DB200PF_PHASE_CLOCK")
    lib.b200pf_phase_clock_read.argtypes = [ctypes.c_void_p, ctypes.c_int]
    buf = np.zeros(N_SLOTS, dtype=np.uint64)

    def read():
        rc = lib.b200pf_phase_clock_read(buf.ctypes.data, N_SLOTS)
        if rc != N_SLOTS:
            raise SystemExit(f"phase_clock.py: reading the counters failed ({rc}): {lib.b200pf_last_error()}")
        return buf.astype(np.float64)

    gm = GridModel.from_npz(os.path.join(GOLD, "gridmodel_l2rpn_case14_sandbox.npz"))
    chron = np.load(os.path.join(GOLD, "case14_sandbox_chronics.npz"))["chron"]
    env = BatchedDoNothing(gm, chron, args.batch)
    eng = env.engine
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    eng.set_stream(stream.cuda_stream)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    for _ in range(max(args.warmup, 3)):
        env.step_device()
    read()
    rows, step_ms = [], []
    for _ in range(args.steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        flush.zero_()
        a.record()
        env.step_device()
        b.record()
        c = read()                              # (synchronises the device)
        step_ms.append(a.elapsed_time(b))
        solves, warps, cycles, ns = c[len(PHASES):]
        if solves <= 0 or warps <= 0 or cycles <= 0:
            raise SystemExit("phase_clock.py: the step did not run the block kernel (no counts)")
        ns_per_cycle = ns / cycles
        us = [c[0] / warps * ns_per_cycle * 1e-3] + [c[k] / solves * ns_per_cycle * 1e-3 for k in range(1, len(PHASES))]
        rows.append(us + [ns / warps * 1e-3, 1e3 / ns_per_cycle])
    rows = np.array(rows)
    med = np.median(rows, axis=0)
    _, _, iters, _ = eng.series_fetch(want_out=False, want_rho=False)
    mean_iters = float(np.mean(iters))
    info = eng.last_launch_info()
    line = {"metric": "block kernel phase clock, l2rpn_case14_sandbox AC, DoNothing, L2 flushed between steps",
            "library": os.path.basename(lib_file), "batch": args.batch, "steps": args.steps, "card": card(),
            "device": torch.cuda.get_device_name(0), "launch": info, "mean_newton_iterations": mean_iters,
            "phases_us_median": {p: round(float(med[k]), 3) for k, p in enumerate(PHASES)},
            "sum_of_phases_us": round(float(med[:len(PHASES)].sum()), 3),
            "warp_span_us_median": round(float(med[len(PHASES)]), 3),
            "sm_mhz_from_clocks": round(float(med[len(PHASES) + 1]), 1),
            "step_ms_median_instrumented": float(np.median(step_ms)),
            "what": WHAT,
            "note": "per warp, averaged over the warps of the step, median over the steps; Newton phases summed over the iterations"}
    print(json.dumps(line), flush=True)
    env.close()


if __name__ == "__main__":
    main()
