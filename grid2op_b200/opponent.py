"""Line-attack opponents for :class:`grid2op_b200.batched_env.BatchedEnv`: the numpy reference path.

Restates, per instance, grid2op's ``OpponentSpace`` (grid2op/Opponent/opponentSpace.py) with ``BaseActionBudget``
(baseActionBudget.py) and one of two opponents that attack one line at a time with ``set_line_status -1``
(``PowerlineSetAction``):

* ``RandomLineOpponent`` (randomLineOpponent.py): a uniform choice among the connected attackable lines;
* ``WeightedRandomOpponent`` (weightedRandomOpponent.py): the attack time is drawn uniformly within ``attack_period`` steps, the
  line with ``p = rho / rho_normalization / sum`` among the connected attackable lines.

Each instance has its own ``np.random.RandomState`` (the opponent's ``space_prng``).  The arithmetic below is numpy's own, on
numpy scalars, as the reference does it: the budget is a float32 until the first charge (float32 - int64 promotes it to float64
under numpy 2) and stays a float64 until the next reset.  The device body (csrc/b200pf_opp.cuh) restates this module; the tests
hold the two to bit equality.

The cost of an attack is ``aff_lines.sum() + aff_subs.sum()`` of ``get_topological_impact``.  For a ``set_line_status -1`` action
on one line that is 1 whatever line status the impact is computed (or was cached) with: the line counts as impacted, no
substation does.  So every step an attack runs costs 1.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

__all__ = ["OPPONENT_KINDS", "BatchedOpponent", "opponent_seed", "NEXT_UNSET"]

OPPONENT_KINDS = {"RandomLineOpponent": 1, "WeightedRandomOpponent": 2}
NEXT_UNSET = -2 ** 31                  # WeightedRandomOpponent._next_attack_time is None (device encoding)
_COST = np.int64(1)                    # BaseActionBudget of one line's set_line_status action


def opponent_seed(env_seed: int) -> int:
    """The opponent's seed after ``env.seed(env_seed)`` (``BaseEnv.seed``, grid2op/Environment/baseEnv.py): the sixth
    ``randint(2**31 - 1)`` of the environment's generator, when chronics, observation space, action space, environment
    modification helper and voltage controller all take one before it (as in every environment ``grid2op.make`` builds)."""
    max_seed = np.iinfo(np.int32).max
    rs = np.random.RandomState(np.array(env_seed).astype(np.int32))
    for _ in range(5):
        rs.randint(max_seed)
    return int(rs.randint(max_seed))


class BatchedOpponent:
    """The opponent state of ``batch`` instances and their random streams (host path)."""

    def __init__(self, kind: str, lines: Sequence[int], batch: int, *, attack_duration: int, attack_cooldown: int,
                 budget_per_ts: float, init_budget: float, seeds, attack_period: Optional[int] = None,
                 rho_normalization: Optional[Sequence[float]] = None):
        if kind not in OPPONENT_KINDS:
            raise ValueError(f"unknown opponent {kind!r} ({' / '.join(OPPONENT_KINDS)})")
        self.kind = kind
        self.code = OPPONENT_KINDS[kind]
        self.lines = np.asarray(lines, dtype=np.int64)
        if self.lines.ndim != 1 or not 1 <= len(self.lines) <= 64:
            raise ValueError("1 to 64 attackable lines")
        self.weighted = kind == "WeightedRandomOpponent"
        if self.weighted:
            if attack_period is None or int(attack_period) <= 0:
                raise ValueError("WeightedRandomOpponent needs attack_period > 0")
            norm = np.ones(len(self.lines)) if rho_normalization is None or len(rho_normalization) == 0 else np.array(rho_normalization, dtype=np.float64)
            if norm.shape != self.lines.shape:
                raise ValueError("rho_normalization must have one value per attacked line")
            self.rho_norm = norm
        else:
            self.rho_norm = np.ones(len(self.lines))
        self.attack_period = int(attack_period) if attack_period is not None else 0
        # grid2op's constructor casts: dt_int durations, dt_float budgets (baseEnv.py)
        self.attack_duration = np.int32(attack_duration)
        self.attack_cooldown = np.int32(attack_cooldown)
        self.budget_per_ts = np.float32(budget_per_ts)
        self.init_budget = np.float32(init_budget)
        if self.init_budget < 0:
            raise ValueError("the initial budget must be >= 0")
        seeds = np.asarray(seeds, dtype=np.int64).reshape(-1)
        if len(seeds) != batch:
            raise ValueError(f"{len(seeds)} seeds for {batch} instances")
        self.batch = int(batch)
        self.rngs = [np.random.RandomState(int(s)) for s in seeds]
        self.budget = [self.init_budget] * batch
        self.duration = np.zeros(batch, dtype=np.int64)
        self.cooldown = np.zeros(batch, dtype=np.int64)
        self.last = np.full(batch, -1, dtype=np.int64)
        self.next_time = [None] * batch
        self.reset(np.arange(batch))

    # ---- OpponentSpace.reset ----------------------------------------------------------------------------------------------
    def reset(self, idx):
        """the random streams continue"""
        for i in np.asarray(idx, dtype=np.int64).reshape(-1):
            self.budget[i] = self.init_budget
            self.duration[i] = 0
            self.cooldown[i] = int(self.attack_cooldown)
            self.last[i] = -1
            self.next_time[i] = None

    # ---- OpponentSpace.attack ---------------------------------------------------------------------------------------------
    def attack(self, line_status: np.ndarray, rho: Optional[np.ndarray], live: np.ndarray):
        """One step of every live instance: ``line_status`` bool [B, n_line] and ``rho`` float32 [B, n_line] of the previous step
        (the observation the opponent sees).  -> (attacked line int32 [B], -1 for none; attack duration int32 [B])"""
        line = np.full(self.batch, -1, dtype=np.int32)
        dur = np.zeros(self.batch, dtype=np.int32)
        for i in np.flatnonzero(live):
            a, d = self._attack_one(int(i), line_status[i], None if rho is None else rho[i])
            line[i], dur[i] = a, d
        return line, dur

    def _attack_one(self, i, status, rho):
        self.budget[i] = self.budget[i] + self.budget_per_ts
        self.duration[i] = max(0, self.duration[i] - 1)
        self.cooldown[i] = max(0, self.cooldown[i] - 1)
        asked = False
        if self.duration[i] > 0:
            attack = int(self.last[i])
            attack = None if attack < 0 else attack
        elif self.cooldown[i] > self.attack_cooldown:
            attack = None
        else:
            asked = True
            attack, duration = self._opponent_attack(i, status, rho)
            if duration is None:
                duration = self.attack_duration
            if duration * self._cost(attack) > self.budget[i]:
                attack = None
            if attack is not None:
                self.duration[i] = duration
                self.cooldown[i] += self.attack_cooldown
        if not asked and self.weighted:
            self.next_time[i] = None                                        # tell_attack_continues
        self.budget[i] = self.budget[i] - self._cost(attack)
        self.last[i] = -1 if attack is None else attack
        return (-1, 0) if attack is None else (attack, int(self.duration[i]))

    @staticmethod
    def _cost(attack):
        return 0 if attack is None else _COST

    def _opponent_attack(self, i, status, rho):
        rng = self.rngs[i]
        if self.weighted:
            if self.next_time[i] is None:
                self.next_time[i] = 1 + rng.randint(self.attack_period)
            self.next_time[i] -= 1
            if self.next_time[i] > 0:
                return None, 0
        st = np.asarray(status, dtype=bool)[self.lines]
        if not st.sum():
            return None, 0
        avail = self.lines[st]
        if not self.weighted:
            return int(rng.choice(avail)), None
        r = np.asarray(rho, dtype=np.float32)[self.lines][st] / self.rho_norm[st]
        s = r.sum()
        if s <= 0.0:
            return None, 0
        return int(rng.choice(avail, p=r / s)), None

    # ---- the state as the device keeps it (b200pf_opp_get_state / b200pf_opp_set_state) ------------------------------------
    def get_state(self):
        """-> dict(budget float64 [B], budget64 uint8 [B], ctr int32 [B, 4], mt uint32 [B, 624], mt_pos int32 [B])"""
        B = self.batch
        ctr = np.empty((B, 4), dtype=np.int32)
        ctr[:, 0], ctr[:, 1], ctr[:, 2] = self.duration, self.cooldown, self.last
        ctr[:, 3] = [NEXT_UNSET if t is None else int(t) for t in self.next_time]
        mt = np.empty((B, 624), dtype=np.uint32)
        pos = np.empty(B, dtype=np.int32)
        for i, r in enumerate(self.rngs):
            st = r.get_state()
            mt[i], pos[i] = st[1], st[2]
        return dict(budget=np.array([float(b) for b in self.budget], dtype=np.float64),
                    budget64=np.array([b.dtype == np.float64 for b in self.budget], dtype=np.uint8), ctr=ctr, mt=mt, mt_pos=pos)

    def set_state(self, s):
        for i in range(self.batch):
            self.budget[i] = np.float64(s["budget"][i]) if s["budget64"][i] else np.float32(s["budget"][i])
            self.rngs[i].set_state(("MT19937", np.asarray(s["mt"][i], dtype=np.uint32), int(s["mt_pos"][i]), 0, 0.0))
        self.duration[:], self.cooldown[:], self.last[:] = s["ctr"][:, 0], s["ctr"][:, 1], s["ctr"][:, 2]
        self.next_time = [None if int(t) == NEXT_UNSET else int(t) for t in s["ctr"][:, 3]]
