"""Agent loop with actions: BatchedEnv.step fed by actions copied to the host, then observe, against BatchedEnv.step_tensors, then
observe, alternating in one process.  Random one-substation and one-line actions drawn on the GPU with a seeded torch generator;
protections off and on; case14 at batch 4096 and l2rpn_neurips_2020_track1 at batch 1024.  A host clock around K steps that end in
a device synchronise, after warm-up.  Prints env.step/s (min / median / max over the repeats), the bytes each path copies per step,
and the card and its power limit read in the same run.

``--vector``: grid2op's native topology action on the tensor path instead.  (1) case14 at batch 4096, protections off: the same
one-substation / one-line actions through the legacy arguments and through the set_bus / set_line_status vectors, the two
environments alternating, to isolate the cost of the wider input; (2) l2rpn_idf_2023 at batch 1024 with its RulesByArea:
multi-substation set_bus / change_bus actions with a few line statuses.

``--ids``: discrete action ids into an ``ActionTable`` on the tensor path, ids drawn on the GPU.  (1) case14 at batch 4096, protections
off, the unitary table (IdToAct's 487 topology actions): the same actions as ids and as the four vectors gathered with torch from
the table, the two environments alternating, to isolate what the id encoding saves against the vector encoding; (2) l2rpn_idf_2023
at batch 1024 with its RulesByArea and the full unitary table (147,260 rows, 214 MB): the cost of row reads scattered over it.

    python scripts/bench_env_tensor.py [--steps 50] [--warmup 5] [--repeats 5] [--vector | --ids]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=20)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:                                    # pragma: no cover
        return f"unknown ({e})"


def draw(env, gen, dev):
    import torch
    B, gm = env.batch, env.gm
    sub = torch.randint(0, gm.n_sub, (B,), generator=gen, device=dev, dtype=torch.int32)
    bus = torch.randint(1, 3, (B, env.max_sub_size), generator=gen, device=dev, dtype=torch.int8)
    size = torch.as_tensor(env.sub_size, device=dev)[sub.long()]
    bus[torch.arange(env.max_sub_size, device=dev)[None, :] >= size[:, None]] = 0
    pick = torch.rand(B, generator=gen, device=dev)
    sub[pick >= 0.5] = -1
    line = torch.randint(0, gm.n_line, (B,), generator=gen, device=dev, dtype=torch.int32)
    line[(pick < 0.5) | (pick >= 0.8)] = -1
    lst = torch.where(torch.rand(B, generator=gen, device=dev) < 0.5, -1, 1).to(torch.int32)
    return sub, bus, line, lst


def run(name, B, protections, steps, warmup, repeats):
    import torch
    from conftest import env_grid
    from grid2op_b200.batched_env import BatchedEnv
    from grid2op_b200.chronics import list_scenarios, load_scenarios
    from grid2op_b200.gridmodel import GridModel
    grid = env_grid(name)
    gm = GridModel(grid)
    env_dir = os.path.dirname(grid)
    folders = list_scenarios(os.path.join(env_dir, "chronics"))[:4]
    chron = load_scenarios(os.path.join(env_dir, "chronics"), gm, scenarios=folders)
    dev = torch.device("cuda", 0)
    envs = {}
    for mode in ("host", "tensor"):
        e = BatchedEnv(gm, chron, B, nb_timestep_cooldown_line=2, nb_timestep_cooldown_sub=2, protections=protections)
        e.enable_observation(env_dir, scenarios=folders)
        if protections:             # (random actions reach more new topologies per step than the automatic policy plans for)
            e.engine.set_kernel_policy(e.engine.KERNEL_PLANNED)
        envs[mode] = e
    gens = {m: torch.Generator(device=dev) for m in envs}
    for m, g in gens.items():
        g.manual_seed(0)

    def one(mode):
        e = envs[mode]
        sub, bus, line, lst = draw(e, gens[mode], dev)
        if mode == "host":
            _, done, _ = e.step(sub.cpu().numpy(), bus.cpu().numpy(), line.cpu().numpy(), lst.cpu().numpy())
            e.observe()
            if done.any():                                    # finished instances restart
                e.reset_instances(np.flatnonzero(done))
        else:
            _, done, _ = e.step_tensors(sub, bus, line, lst)
            e.observe()
            e.reset_instances(done.clone())

    topo_up = [0]
    orig = envs["host"].engine.series_set_topo

    def set_topo(topo):
        topo_up[0] += 1
        return orig(topo)
    envs["host"].engine.series_set_topo = set_topo

    def timed(mode):
        for _ in range(warmup):
            one(mode)
        torch.cuda.synchronize()
        s0 = envs[mode].engine.env_stats() if mode == "tensor" else None
        o0 = envs[mode].engine.obs_stats()
        topo_up[0] = 0
        t0 = time.perf_counter()
        for _ in range(steps):
            one(mode)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        o1 = envs[mode].engine.obs_stats()
        if mode == "tensor":
            s1 = envs[mode].engine.env_stats()
            h2d, d2h = s1["h2d_bytes"] - s0["h2d_bytes"], s1["d2h_bytes"] - s0["d2h_bytes"] + o1["d2h_bytes"] - o0["d2h_bytes"]
        else:                      # observe inputs + series fetches; the topology uploads are added below
            h2d, d2h = o1["h2d_bytes"] - o0["h2d_bytes"], o1["d2h_bytes"] - o0["d2h_bytes"]
            h2d += topo_up[0] * envs[mode].gm.n_topo_in * B
            topo_up[0] = 0
        return B * steps / dt, h2d / steps, d2h / steps

    res = {m: [] for m in envs}
    envs["host"].reset_step(); envs["tensor"].step_tensors(from_reset=True)
    for _ in range(repeats):
        for m in ("host", "tensor"):
            res[m].append(timed(m))
    for m in ("host", "tensor"):
        r = np.array([x[0] for x in res[m]])
        print(f"{name:28s} B={B:5d} prot={int(protections)} {m:6s}: env.step/s min {r.min():.3e} median {np.median(r):.3e} max {r.max():.3e}; "
              f"per step H2D {res[m][-1][1] / 1e3:.1f} kB, "
              f"D2H {res[m][-1][2] / 1e3:.1f} kB")
    for e in envs.values():
        e.close()


def as_vectors(env, sub, bus, line, lst):
    """the one-substation / one-line action as set_bus int8 [B, dim_topo] / set_line_status int8 [B, n_line], on the device"""
    import torch
    B, gm, dev = env.batch, env.gm, sub.device
    pos = torch.as_tensor(env.sub_pos, device=dev)[sub.clamp(min=0).long()]                  # [B, max_sub]
    ok = (pos >= 0) & (sub[:, None] >= 0) & (bus > 0)
    sb = torch.zeros((B, gm.dim_topo + 1), dtype=torch.int8, device=dev)                    # (last column: dump for padding)
    sb.scatter_(1, torch.where(ok, pos, gm.dim_topo), torch.where(ok, bus, 0))
    ss = torch.zeros((B, gm.n_line + 1), dtype=torch.int8, device=dev)
    ss.scatter_(1, torch.where(line >= 0, line, gm.n_line).long()[:, None], lst.to(torch.int8)[:, None])
    return sb[:, :gm.dim_topo].contiguous(), ss[:, :gm.n_line].contiguous()


def draw_multi(env, gen, dev):
    """several substations per instance set or changed, and a few line statuses set (idf_2023: up to three of each are legal)"""
    import torch
    B, gm = env.batch, env.gm
    sub_of = torch.as_tensor(env.sub_of_pos, device=dev)
    pick = torch.rand((B, gm.n_sub), generator=gen, device=dev) < 3.0 / gm.n_sub
    touched = pick[:, sub_of] & (torch.rand((B, gm.dim_topo), generator=gen, device=dev) < 0.5)
    use_set = (torch.rand((B, gm.n_sub), generator=gen, device=dev) < 0.5)[:, sub_of]
    two = torch.rand((B, gm.dim_topo), generator=gen, device=dev) < 0.3
    sb = torch.where(touched & use_set, torch.where(two, 2, 1), 0).to(torch.int8)
    cb = touched & ~use_set & two
    ss = torch.where(torch.rand((B, gm.n_line), generator=gen, device=dev) < 1.0 / gm.n_line,
                     torch.where(torch.rand((B, gm.n_line), generator=gen, device=dev) < 0.5, -1, 1), 0).to(torch.int8)
    return sb, cb, ss


def run_vector(name, B, steps, warmup, repeats, modes, rules_by_area=None):
    """``modes``: ("legacy", "vector") for the same one-substation actions in the two encodings, ("multi",), or ("ids", "rows")
    / ("ids",) for ids into the unitary action table and the same rows as vectors"""
    import torch
    from conftest import env_grid
    from grid2op_b200.batched_env import BatchedEnv
    from grid2op_b200.chronics import list_scenarios, load_scenarios
    from grid2op_b200.gridmodel import GridModel
    grid = env_grid(name)
    gm = GridModel(grid)
    env_dir = os.path.dirname(grid)
    folders = list_scenarios(os.path.join(env_dir, "chronics"))[:4]
    chron = load_scenarios(os.path.join(env_dir, "chronics"), gm, scenarios=folders)
    dev = torch.device("cuda", 0)
    table = tab = None
    if "ids" in modes or "rows" in modes:
        from grid2op_b200.action_table import ActionTable
        table = ActionTable.unitary(gm)
        tab = [torch.as_tensor(np.array(x), device=dev) for x in (table.set_bus, table.change_bus, table.set_line_status,
                                                                     table.change_line_status)]
        print(f"{name}: action table of {table.n} rows, {sum(x.numel() for x in tab) / 1e6:.1f} MB")
    envs, gens = {}, {}
    for mode in modes:
        e = BatchedEnv(gm, chron, B, nb_timestep_cooldown_line=2, nb_timestep_cooldown_sub=2, protections=False,
                       rules_by_area=rules_by_area, max_sub_changed=1 if rules_by_area else 3, max_line_status_changed=1 if rules_by_area else 2)
        e.enable_observation(env_dir, scenarios=folders)
        if mode == "ids":
            e.set_action_table(table)
        envs[mode] = e
        gens[mode] = torch.Generator(device=dev)
        gens[mode].manual_seed(0)

    def one(mode):
        e = envs[mode]
        if mode == "multi":
            sb, cb, ss = draw_multi(e, gens[mode], dev)
            _, done, _ = e.step_tensors(set_bus=sb, change_bus=cb, set_line_status=ss)
        elif mode in ("ids", "rows"):
            ids = torch.randint(0, table.n, (B,), generator=gens[mode], device=dev, dtype=torch.int32)
            if mode == "ids":
                _, done, _ = e.step_tensors(action_id=ids)
            else:
                _, done, _ = e.step_tensors(set_bus=tab[0][ids], change_bus=tab[1][ids], set_line_status=tab[2][ids],
                                            change_line_status=tab[3][ids])
        else:
            sub, bus, line, lst = draw(e, gens[mode], dev)
            if mode == "legacy":
                _, done, _ = e.step_tensors(sub, bus, line, lst)
            else:
                sb, ss = as_vectors(e, sub, bus, line, lst)
                _, done, _ = e.step_tensors(set_bus=sb, set_line_status=ss)
        e.observe()
        e.reset_instances(done.clone())

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
        return (B * steps / dt, (s1["h2d_bytes"] - s0["h2d_bytes"]) / steps,
                (s1["d2h_bytes"] - s0["d2h_bytes"] + o1["d2h_bytes"] - o0["d2h_bytes"]) / steps, (s1["host_waits"] - s0["host_waits"]) / steps)

    for e in envs.values():
        e.step_tensors(from_reset=True)
    res = {m: [] for m in envs}
    for _ in range(repeats):
        for m in modes:
            res[m].append(timed(m))
    for m in modes:
        r = np.array([x[0] for x in res[m]])
        print(f"{name:28s} B={B:5d} {m:6s}: env.step/s min {r.min():.3e} median {np.median(r):.3e} max {r.max():.3e}; per step H2D "
              f"{res[m][-1][1] / 1e3:.1f} kB, D2H {res[m][-1][2] / 1e3:.1f} kB, host waits {res[m][-1][3]:.2f}")
    for e in envs.values():
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--vector", action="store_true")
    ap.add_argument("--ids", action="store_true")
    args = ap.parse_args()
    print("card, power limit:", card())
    if args.ids:
        from test_env_actions_gpu import _idf_rule_areas
        run_vector("l2rpn_case14_sandbox", 4096, args.steps, args.warmup, args.repeats, ("ids", "rows"))
        run_vector("l2rpn_idf_2023", 1024, args.steps, args.warmup, args.repeats, ("ids",), rules_by_area=_idf_rule_areas())
        return
    if args.vector:
        from test_env_actions_gpu import _idf_rule_areas
        run_vector("l2rpn_case14_sandbox", 4096, args.steps, args.warmup, args.repeats, ("legacy", "vector"))
        run_vector("l2rpn_idf_2023", 1024, args.steps, args.warmup, args.repeats, ("multi",), rules_by_area=_idf_rule_areas())
        return
    for name, B in (("l2rpn_case14_sandbox", 4096), ("l2rpn_neurips_2020_track1", 1024)):
        for prot in (False, True):
            run(name, B, prot, args.steps, args.warmup, args.repeats)


if __name__ == "__main__":
    main()
