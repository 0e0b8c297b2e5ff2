"""grid2op's alarms (l2rpn_icaps_2021) for a whole batch, on the host: the zones, the environment's attention budget and the
AlarmReward.

Reference (grid2op 1.12.5), per environment:

* ``BaseEnv.load_alarm_data`` (grid2op/Environment/baseEnv.py:1057-1126): the ``"fixed"`` zones of ``alerts_info.json``, sorted by
  name; a line may be in several zones, every line must be in one;
* ``LinearAttentionBudget`` (grid2op/operator_attention/attention_budget.py): ``register_action`` in ``BaseEnv.step`` once the
  action's legality is known (baseEnv.py:3769-3775), ``reset`` at ``env.reset()``;
* ``AlarmReward`` (grid2op/Reward/alarmReward.py), the environment's reward class: non-zero only on the step that ends the
  episode; its ``is_alarm_used``, which no reset clears, is what the game-over observation shows as
  ``was_alarm_used_after_game_over``.

AlarmReward scores only the successful alarms of the last ``best_time + window_size`` steps, so :class:`BatchedAlarms` keeps a
ring of that many (step, zone mask) entries per instance instead of ``_all_successful_alarms``, and a flag "this episode had a
successful alarm".  It keeps the same arrays as the device (csrc/b200pf_alarm.cuh, ``b200pf_alarm_get_state``) so that the two
paths hand the state over as it is.
"""
from __future__ import annotations

import json
import os
from typing import Dict, List, Tuple

import numpy as np

__all__ = ["BatchedAlarms", "ALARM_STATE", "MAX_ZONES", "MAX_RING", "load_alarm_zones"]

MAX_ZONES = 32            # one bit per zone in a uint32 mask
MAX_RING = 1024           # best_time + window_size: the ring of successful alarms an instance keeps

# the state arrays in the order of b200pf_alarm_get_state / _set_state
ALARM_STATE = (("budget", np.float32), ("time_last", np.int32), ("time_last_ok", np.int32), ("last", np.int32), ("last_ok", np.int32),
               ("ring_step", np.int32), ("ring_mask", np.uint32), ("any_ok", np.uint8), ("used", np.uint8), ("illegal", np.uint8))


def load_alarm_zones(env_dir: str, gm) -> Tuple[List[str], np.ndarray]:
    """-> (zone names, sorted; uint32 [n_line] zones of every line, bit z for zone z) from the ``"fixed"`` key of
    ``env_dir/alerts_info.json``, as ``BaseEnv.load_alarm_data`` reads it.  ValueError where grid2op raises EnvError (a line
    unknown to the grid, a line in no zone, a file with neither key), for a missing file or a file without ``"fixed"`` (no
    alarms), and for more than 32 zones."""
    path = os.path.join(env_dir, "alerts_info.json")
    if not os.path.isfile(path):
        raise ValueError(f"{path}: no alerts_info.json, the environment has no alarms")
    with open(path, encoding="utf-8") as f:
        d = json.load(f)
    if "fixed" not in d:
        raise ValueError(f"{path}: no \"fixed\" zones (line alerts or nothing), the environment has no alarms")
    names = sorted(d["fixed"].keys())
    if len(names) > MAX_ZONES:
        raise ValueError(f"{len(names)} alarm zones, at most {MAX_ZONES}")
    line_names = list(gm.name_line)
    index = {nm: i for i, nm in enumerate(line_names)}
    mask = np.zeros(gm.n_line, dtype=np.uint32)
    for z, zone in enumerate(names):
        for line in d["fixed"][zone]:
            if line not in index:
                raise ValueError(f"{path}: line {line!r} of zone {zone!r} is not in the grid")
            mask[index[line]] |= np.uint32(1 << z)
    if (mask == 0).any():
        raise ValueError(f"{path}: line {line_names[int(np.flatnonzero(mask == 0)[0])]!r} is in no zone")
    return names, mask


class BatchedAlarms:
    def __init__(self, zone_mask, n_zone: int, batch: int, *, max_budget=3.0, budget_per_ts=1.0 / 192, alarm_cost=1.0, init_budget=2.0,
                 best_time: int = 12, window_size: int = 12, reward: bool = True):
        self.zone_mask = np.ascontiguousarray(zone_mask, dtype=np.uint32)
        self.n, self.batch = int(n_zone), int(batch)
        self.best_time, self.window = int(best_time), int(window_size)
        self.ring, self.reward = self.best_time + self.window, bool(reward)
        f = np.float32
        # LinearAttentionBudget.init: float32 constants
        self.max_budget, self.budget_per_ts, self.alarm_cost, self.init_budget = f(max_budget), f(budget_per_ts), f(alarm_cost), f(init_budget)
        B, n, R = self.batch, self.n, self.ring
        shapes = dict(last=(B, n), last_ok=(B, n), ring_step=(B, R), ring_mask=(B, R))
        self.s: Dict[str, np.ndarray] = {k: np.zeros(shapes.get(k, (B,)), dtype=dt) for k, dt in ALARM_STATE}
        self.reward_out = np.zeros(B, dtype=np.float64)
        self.reset(np.arange(B))

    def reset(self, idx):
        """``LinearAttentionBudget.reset`` of the instances ``idx`` (AlarmReward's is_alarm_used is kept)"""
        s = self.s
        s["budget"][idx] = self.init_budget
        for k in ("time_last", "time_last_ok", "last", "last_ok"):
            s[k][idx] = -1
        for k in ("ring_step", "ring_mask", "any_ok", "illegal"):
            s[k][idx] = 0
        self.reward_out[idx] = 0.0

    def step(self, raise_alarm, live, is_illegal, step_no, game_over, disc):
        """one ordinary step: ``raise_alarm`` bool [B, n] (None: no alarm), ``live`` bool [B] (not finished before the step, and not
        a reset step), ``is_illegal`` bool [B] (the agent's action), ``step_no`` int [B] (nb_time_step of the step), ``game_over``
        bool [B] (the step ended the episode with an error), ``disc`` int [B, n_line] (the step's disc_lines; None: protections
        off).  Registers the alarms of the live instances and returns the AlarmReward of every instance (0 for the others)."""
        s, B, n = self.s, self.batch, self.n
        up = np.zeros((B, n), bool) if raise_alarm is None else np.asarray(raise_alarm, dtype=bool).reshape(B, n)
        step_no = np.asarray(step_no, dtype=np.int32)
        act = np.asarray(live, dtype=bool) & ~np.asarray(is_illegal, dtype=bool)
        m = (up.astype(np.uint32) << np.arange(n, dtype=np.uint32)).sum(axis=1, dtype=np.uint32)
        s["illegal"][:] = 0
        b = s["budget"]
        quiet = act & (m == 0)                                 # min(max_budget, budget_per_ts + current), in float32
        nb = self.budget_per_ts + b[quiet]
        b[quiet] = np.where(nb < self.max_budget, nb, self.max_budget)
        has = act & (m != 0)
        s["time_last"][has] = step_no[has]
        rows = has[:, None] & up
        s["last"][rows] = np.broadcast_to(step_no[:, None], (B, n))[rows]
        ok = has & (b >= self.alarm_cost)                      # one charge, whatever the number of zones
        b[ok] = b[ok] - self.alarm_cost
        s["time_last_ok"][ok] = step_no[ok]
        rows = ok[:, None] & up
        s["last_ok"][rows] = np.broadcast_to(step_no[:, None], (B, n))[rows]
        ii = np.flatnonzero(ok)
        slot = step_no[ii] % self.ring
        s["ring_step"][ii, slot] = step_no[ii]
        s["ring_mask"][ii, slot] = m[ii]
        s["any_ok"][ok] = 1
        s["illegal"][has & ~ok] = 1                            # NotEnoughAttentionBudget
        self.reward_out[:] = 0.0
        if self.reward:
            for i in np.flatnonzero(np.asarray(live, dtype=bool) & np.asarray(game_over, dtype=bool)):
                self.reward_out[i] = self._reward_instance(i, int(step_no[i]), None if disc is None else np.asarray(disc)[i])
        return self.reward_out

    def _reward_instance(self, i, step, disc):
        """AlarmReward.__call__ of instance i on the step that ended its episode with an error"""
        s = self.s
        if disc is None or (disc == -1).all() or not s["any_ok"][i]:
            return -1.0                                        # (is_alarm_used left as it was)
        first = np.bitwise_or.reduce(self.zone_mask[disc == 0], initial=np.uint32(0))
        W, bt = self.window, self.best_time
        best = -1.0
        for sa, m in zip(s["ring_step"][i].tolist(), s["ring_mask"][i].tolist()):
            dist = step - sa
            if sa <= 0 or not 0 <= dist < self.ring or dist > bt + W or dist < bt - W:
                continue
            d = dist - bt
            t = float(-((d - W) * (d + W))) / float(W * W)
            if t == 0.0:                                       # at either end of the window: reward_min, not used
                continue
            sc = t * (1.0 if bin(m).count("1") == 1 and m & int(first) else 0.5)
            if sc > best:
                best = sc
        s["used"][i] = best > -1.0
        return best

    def obs_record(self, current_step) -> np.ndarray:
        """int32 [B, n + 4]: the alarm values of the observe input record (alarm_obs_record of csrc/b200pf_alarm.cuh)"""
        s = self.s
        tok = s["time_last_ok"]
        tsl = np.where(tok > 0, np.asarray(current_step, dtype=np.int32) - tok, -1)
        return np.concatenate([s["illegal"][:, None], tsl[:, None], s["last_ok"], s["budget"].view(np.int32)[:, None],
                               s["used"][:, None]], axis=1).astype(np.int32)

    def get_state(self) -> Dict[str, np.ndarray]:
        return {k: v.copy() for k, v in self.s.items()}

    def set_state(self, st: Dict[str, np.ndarray]):
        for k, dt in ALARM_STATE:
            self.s[k][:] = np.asarray(st[k], dtype=dt).reshape(self.s[k].shape)
