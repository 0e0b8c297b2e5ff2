#!/usr/bin/env python
"""Cost of the observation layer (``BatchedEnv.observe``, csrc/b200pf_obs.cuh) next to the series step it follows, on the GPU.

l2rpn_case14_sandbox AC, DoNothing, batch 4096 (the workload of bench.py): every timed iteration is one series step, and every
other one also enqueues the observe launch behind it (full CompleteObservation vector + RedispReward into torch tensors, after the
H2D of the per-instance host inputs), alternating so that both variants see the same clocks.  CUDA events on the launching stream,
L2 flushed between iterations (outside the event pairs) like bench.py.  The static tables are synthetic (zero calendar, made-up
generator costs): the kernel's work does not depend on their values.  Prints one JSON line; writes nothing.

    python scripts/bench_observe.py [--steps 200] [--warmup 10] [--batch 4096]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
GOLD = os.path.join(REPO, "tests", "golden")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200, help="timed iterations of each variant")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--batch", type=int, default=4096)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_observe.py: no CUDA device (this measurement has no CPU fallback)")
    from grid2op_b200.gridmodel import GridModel
    from grid2op_b200.observation import obs_spec
    from grid2op_b200.rollout import BatchedDoNothing
    gm = GridModel.from_npz(os.path.join(GOLD, "gridmodel_l2rpn_case14_sandbox.npz"))
    chron = np.load(os.path.join(GOLD, "case14_sandbox_chronics.npz"))["chron"]
    B = args.batch
    env = BatchedDoNothing(gm, chron, B)
    eng = env.engine
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    eng.set_stream(stream.cuda_stream)
    seg, n_obs = obs_spec(gm)
    ng = gm.n_gen
    gen = dict(gen_pmin=np.zeros(ng, np.float32), gen_pmax=np.full(ng, 100.0, np.float32), gen_max_ramp_up=np.full(ng, 5.0, np.float32),
               gen_max_ramp_down=np.full(ng, 5.0, np.float32), gen_cost_per_MW=np.arange(1, ng + 1, dtype=np.float32),
               gen_renewable=np.zeros(ng, bool), available=True)
    eng.obs_bind(dict(seg=seg, n_obs=n_obs, calendar=np.zeros(chron.shape[:2] + (6,), np.int32),
                      max_step=np.full(chron.shape[0], chron.shape[1] - 1), delta_time=5.0, gen=gen,
                      storage=dict(charge0=np.zeros(gm.n_storage, np.float32), loss_step=np.zeros(gm.n_storage, np.float32)),
                      reward_kind=1, reward=dict(max_regret=1000.0, reward_min=-10.0, reward_illegal=0.0, dts_hours=5 / 60), soft_thr=1.0))
    obs_t = torch.empty((B, n_obs), dtype=torch.float32, device="cuda")
    rew_t = torch.empty((B,), dtype=torch.float32, device="cuda")
    host_in = np.zeros((B, gm.n_line + gm.n_sub + 3), dtype=np.int32)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    k = [0]

    def step(with_obs, mark=None):
        env.step_device()
        if with_obs:
            if mark is not None:
                mark.record()
            host_in[:, -2] = k[0]
            eng.observe(host_in, obs_t.data_ptr(), rew_t.data_ptr())
        k[0] += 1

    for i in range(max(args.warmup, 3)):
        step(i % 2 == 1)
    torch.cuda.synchronize()
    ev = {v: [] for v in (False, True)}
    for i in range(2 * args.steps):
        with_obs = i % 2 == 1
        a, m, b = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        flush.zero_()
        a.record()
        step(with_obs, m)
        b.record()
        ev[with_obs].append((a, m, b))
    torch.cuda.synchronize()
    plain = np.array([a.elapsed_time(b) for a, _, b in ev[False]])
    full = np.array([a.elapsed_time(b) for a, _, b in ev[True]])
    tail = np.array([m.elapsed_time(b) for _, m, b in ev[True]])
    st = eng.obs_stats()
    ok = bool(torch.isfinite(obs_t).all().item() and torch.isfinite(rew_t).all().item())
    line = {"metric": "observe launch cost per step, l2rpn_case14_sandbox AC, DoNothing", "batch": B, "n_obs": n_obs, "steps": args.steps,
            "card": card(), "device": torch.cuda.get_device_name(0),
            "ms_step_median": float(np.median(plain)), "ms_step_plus_observe_median": float(np.median(full)),
            "ms_observe_median": float(np.median(tail)), "ms_observe_mean": float(tail.mean()),
            "ms_observe_spread": [float(tail.min()), float(tail.max())],
            "bytes_written_per_step": st["bytes_written_per_launch"], "h2d_bytes_per_step": st["h2d_bytes"] // max(st["launches"], 1),
            "outputs_finite": ok,
            "what": "ms_observe = CUDA events from the end of the step's solve to the end of the observe launch (H2D of the host inputs + "
                    "the launch); ms_step = the step alone, alternating iterations of the same run"}
    print(json.dumps(line), flush=True)
    env.close()


if __name__ == "__main__":
    main()
