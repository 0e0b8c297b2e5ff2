"""BatchedEnv.step_tensors with and without the line-attack opponent (enable_opponent), alternating in one process, on the workloads
of scripts/bench_env_tensor.py: random one-substation and one-line actions drawn on the GPU with a seeded torch generator, then
observe, finished instances reset on the device; protections off and on; case14 at batch 4096 (RandomLineOpponent on the lines of
rte_case14_opponent), l2rpn_neurips_2020_track1 at batch 1024 (its WeightedRandomOpponent) and l2rpn_wcci_2022_dev at batch 1024
(its GeometricOpponent, with the environment's own constants: its device resets draw a new attack schedule) and l2rpn_idf_2023 at
batch 1024 (its GeometricOpponentMultiArea, three areas, with its own constants).  The first two use their
environments' constants with a small initial budget, so that attacks run from the first steps on.  A host clock around K steps that end in a device
synchronise, after warm-up.  Prints env.step/s (min / median / max over the repeats), the extra bytes per step the opponent moves, and
the card and its power limit read in the same run.

With ``--alerts``: l2rpn_idf_2023 at batch 1024 with its multi-area opponent in both runs, protections off, line alerts off and
on (``enable_alerts`` on the opponent's 22 lines, a random alert tensor drawn on the GPU every step), alternating in one process.

With ``--alarms``: l2rpn_icaps_2021 at batch 1024 with its GeometricOpponent in both runs, protections off and on, alarms off and on
(``enable_alarms`` on the environment's three zones, a random alarm tensor drawn on the GPU every step), alternating in one process.

    python scripts/bench_opponent.py [--steps 50] [--warmup 5] [--repeats 5] [--alerts] [--alarms]
"""
import argparse
import os
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "scripts"))

OPPONENTS = {
    "l2rpn_case14_sandbox": dict(kind="RandomLineOpponent", lines=["1_3_3", "1_4_4", "3_6_15", "9_10_12", "11_12_13", "12_13_14"],
                                 attack_duration=48, attack_cooldown=288, budget_per_ts=0.5, init_budget=48.0),
    "l2rpn_neurips_2020_track1": dict(kind="WeightedRandomOpponent",
                                      lines=["62_58_180", "62_63_160", "48_50_136", "48_53_141", "41_48_131", "39_41_121", "43_44_125",
                                             "44_45_126", "34_35_110", "54_58_154"],
                                      rho_normalization=[0.45, 0.45, 0.6, 0.35, 0.3, 0.2, 0.55, 0.3, 0.45, 0.55], attack_period=12,
                                      attack_duration=48, attack_cooldown=288, budget_per_ts=0.16667, init_budget=48.0),
    # the environment's own GeometricOpponent (config.py): attacks every 24 h on average, 4 h long, at least 1 h
    "l2rpn_wcci_2022_dev": dict(kind="GeometricOpponent",
                                lines=["26_31_106", "21_22_93", "17_18_88", "4_10_162", "12_14_68", "14_32_108", "62_58_180", "62_63_160",
                                       "48_50_136", "48_53_141", "41_48_131", "39_41_121", "43_44_125", "44_45_126", "34_35_110",
                                       "54_58_154", "74_117_81", "80_79_175", "93_95_43", "88_91_33", "91_92_37", "99_105_62",
                                       "102_104_61"],
                                attack_duration=96, attack_cooldown=12, budget_per_ts=0.17, init_budget=144.0, attack_every_xxx_hour=24,
                                average_attack_duration_hour=4, minimum_attack_duration_hour=1),
    # the environment's own GeometricOpponentMultiArea (config.py): three areas, attacks every 32 h on average, 2 h long, at least 1 h
    "l2rpn_idf_2023": dict(kind="GeometricOpponentMultiArea",
                           lines=[["26_31_106", "21_22_93", "17_18_88", "4_10_162", "12_14_68", "29_37_117"],
                                  ["62_58_180", "62_63_160", "48_50_136", "48_53_141", "41_48_131", "39_41_121", "43_44_125", "44_45_126",
                                   "34_35_110", "54_58_154"],
                                  ["74_117_81", "93_95_43", "88_91_33", "91_92_37", "99_105_62", "102_104_61"]],
                           attack_duration=96, attack_cooldown=0, budget_per_ts=0.51, init_budget=1000.0, attack_every_xxx_hour=32,
                           average_attack_duration_hour=2, minimum_attack_duration_hour=1),
    # the environment's own GeometricOpponent (config.py): attacks every 24 h on average, 4 h long, at least 1 h
    "l2rpn_icaps_2021": dict(kind="GeometricOpponent",
                             lines=["62_58_180", "62_63_160", "48_50_136", "48_53_141", "41_48_131", "39_41_121", "43_44_125", "44_45_126",
                                    "34_35_110", "54_58_154"],
                             attack_duration=96, attack_cooldown=12, budget_per_ts=0.17, init_budget=144.0, attack_every_xxx_hour=24,
                             average_attack_duration_hour=4, minimum_attack_duration_hour=1),
}


def run(name, B, protections, steps, warmup, repeats, alerts=False, alarms=False):
    """``alerts`` / ``alarms``: both environments run the opponent, the second one also the line alerts / the alarms (the comparison
    is alerts / alarms off against on)"""
    import torch
    from bench_env_tensor import draw
    from conftest import env_grid
    from grid2op_b200.batched_env import BatchedEnv
    from grid2op_b200.chronics import list_scenarios, load_scenarios
    from grid2op_b200.gridmodel import GridModel
    from grid2op_b200.opponent import opponent_seed
    from grid2op_b200.alarm import load_alarm_zones
    grid = env_grid(name)
    gm = GridModel(grid)
    env_dir = os.path.dirname(grid)
    folders = list_scenarios(os.path.join(env_dir, "chronics"))[:4]
    chron = load_scenarios(os.path.join(env_dir, "chronics"), gm, scenarios=folders)
    dev = torch.device("cuda", 0)
    envs = {}
    for mode in ("off", "on"):
        e = BatchedEnv(gm, chron, B, nb_timestep_cooldown_line=2, nb_timestep_cooldown_sub=2, protections=protections)
        if alerts and mode == "on":
            e.enable_alerts(OPPONENTS[name]["lines"])
        if alarms and mode == "on":
            e.enable_alarms(load_alarm_zones(env_dir, gm))
        e.enable_observation(env_dir, scenarios=folders)
        if protections:
            e.engine.set_kernel_policy(e.engine.KERNEL_PLANNED)
        e.step_tensors(from_reset=True)
        if mode == "on" or alerts or alarms:
            o = dict(OPPONENTS[name])
            e.enable_opponent(o.pop("kind"), o.pop("lines"), seeds=[opponent_seed(s) for s in range(B)], **o)
        envs[mode] = e
    gens = {m: torch.Generator(device=dev) for m in envs}
    for g in gens.values():
        g.manual_seed(0)
    attacks = {m: 0 for m in envs}

    n_alert = envs["on"]._alerts.n if alerts else 0
    n_alarm = envs["on"]._alarms.n if alarms else 0

    def one(mode, count=False):
        e = envs[mode]
        act = draw(e, gens[mode], dev)
        if mode == "on" and alerts:              # (drawn in both modes, so that both streams draw the same actions)
            up = torch.rand((B, n_alert), device=dev, generator=gens[mode]) < 0.3
            _, done, info = e.step_tensors(*act, raise_alert=up)
        elif mode == "on" and alarms:
            up = torch.rand((B, n_alarm), device=dev, generator=gens[mode]) < 0.05
            _, done, info = e.step_tensors(*act, raise_alarm=up)
        else:
            if alerts or alarms:
                torch.rand((B, n_alert or n_alarm), device=dev, generator=gens[mode])
            _, done, info = e.step_tensors(*act)
        e.observe()
        e.reset_instances(done.clone())
        if count and "opponent_attack_line" in info:
            attacks[mode] += int((info["opponent_attack_line"] >= 0).reshape(B, -1).any(1).sum())

    def timed(mode):
        for _ in range(warmup):
            one(mode)
        torch.cuda.synchronize()
        s0, o0 = envs[mode].engine.env_stats(), envs[mode].engine.obs_stats()
        t0 = time.perf_counter()
        for _ in range(steps):
            one(mode)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        s1, o1 = envs[mode].engine.env_stats(), envs[mode].engine.obs_stats()
        moved = (s1["h2d_bytes"] - s0["h2d_bytes"]) + (s1["d2h_bytes"] - s0["d2h_bytes"]) + (o1["d2h_bytes"] - o0["d2h_bytes"])
        return B * steps / dt, moved / steps

    res = {m: [] for m in envs}
    for _ in range(repeats):
        for m in ("off", "on"):
            res[m].append(timed(m))
    one("on", count=True)
    for m in ("off", "on"):
        r = np.array([x[0] for x in res[m]])
        print(f"{name:28s} B={B:5d} prot={int(protections)} {'alerts' if alerts else 'alarms' if alarms else 'opponent'} {m:3s}: env.step/s min {r.min():.3e} median {np.median(r):.3e} "
              f"max {r.max():.3e}; bytes moved per step {np.median([x[1] for x in res[m]]) / 1e3:.1f} kB")
    print(f"{'':28s} attacks running in the last step: {attacks['on']} of {B}")
    for e in envs.values():
        e.close()


def main():
    from bench_env_tensor import card
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--only", default=None, help="one workload (environment name)")
    ap.add_argument("--alerts", action="store_true", help="l2rpn_idf_2023 with its opponent, line alerts off / on")
    ap.add_argument("--alarms", action="store_true", help="l2rpn_icaps_2021 with its opponent, alarms off / on")
    args = ap.parse_args()
    print("card, power limit:", card())
    if args.alerts:
        run("l2rpn_idf_2023", 1024, False, args.steps, args.warmup, args.repeats, alerts=True)
        return
    if args.alarms:
        for prot in (False, True):
            run("l2rpn_icaps_2021", 1024, prot, args.steps, args.warmup, args.repeats, alarms=True)
        return
    for name, B in (("l2rpn_case14_sandbox", 4096), ("l2rpn_neurips_2020_track1", 1024), ("l2rpn_wcci_2022_dev", 1024),
                    ("l2rpn_idf_2023", 1024)):
        if args.only and name != args.only:
            continue
        for prot in (False, True):
            run(name, B, prot, args.steps, args.warmup, args.repeats)


if __name__ == "__main__":
    main()
