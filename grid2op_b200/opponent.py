"""Line-attack opponents for :class:`grid2op_b200.batched_env.BatchedEnv`: the numpy reference path.

Restates, per instance, grid2op's ``OpponentSpace`` (grid2op/Opponent/opponentSpace.py) with ``BaseActionBudget``
(baseActionBudget.py) and one of two opponents that attack one line at a time with ``set_line_status -1``
(``PowerlineSetAction``):

* ``RandomLineOpponent`` (randomLineOpponent.py): a uniform choice among the connected attackable lines;
* ``WeightedRandomOpponent`` (weightedRandomOpponent.py): the attack time is drawn uniformly within ``attack_period`` steps, the
  line with ``p = rho / rho_normalization / sum`` among the connected attackable lines;
* ``GeometricOpponent`` (geometricOpponent.py): at every reset it draws a schedule for the whole episode, geometric waiting times
  and durations (``RandomState.geometric``); an attack whose time has come is consumed, and lands only when every attackable line
  is connected (grid2op's ``~status.all()`` test), on a line drawn with Boltzmann weights ``exp(b_beta * rank)`` of the lines'
  rho ranks, for the schedule's duration.  OpponentSpace refuses it (and sets ``previous_fails``, which moves the next attack) when
  that duration exceeds ``attack_duration`` or the budget.  Ranks of equal rho follow the line order (a stable argsort): numpy's
  default argsort is not stable for ties on every host, so that is the one place the reference's own choice can differ;
* ``GeometricOpponentMultiArea`` (geometricOpponentMultiArea.py): one GeometricOpponent per area of lines, each with its own
  ``RandomState`` (seeded by ``randint(2**31 - 1)`` draws of the multi-area opponent's own stream, in area order), schedule and
  ``_next_attack_time``.  Every step, each area's counter ticks down (clamped at -1); an area at -1 asks its GeometricOpponent
  (``~status.all()``, ranks and ``b_beta`` over its own lines, OpponentSpace's shared ``previous_fails``), remembers the line and
  counts the attack's duration, an area still counting repeats its remembered line.  The combined attack has duration 1 and costs
  its line count; OpponentSpace refuses it whole when that exceeds the budget, and the counters stay.  With duration 1 and an
  ``attack_cooldown`` of 0 or 1 OpponentSpace asks on every step; a larger cooldown makes it skip a step and call the multi-area
  ``tell_attack_continues``, which raises in grid2op, so such configurations are refused here.

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

__all__ = ["OPPONENT_KINDS", "BatchedOpponent", "opponent_seed", "geometric_constants", "NEXT_UNSET", "MAX_AREAS", "MULTI_KEYS"]

OPPONENT_KINDS = {"RandomLineOpponent": 1, "WeightedRandomOpponent": 2, "GeometricOpponent": 3, "GeometricOpponentMultiArea": 4}
NEXT_UNSET = -2 ** 31                  # WeightedRandomOpponent / GeometricOpponent._next_attack_time is None (device encoding)
MAX_AREAS = 8                          # GeometricOpponentMultiArea: the device keeps fixed-size per-instance arrays
# GeometricOpponentMultiArea's per-area counters (multi_ctr [B, n_area, 6]): schedule length, attacks consumed, _next_attack_time,
# entries dropped at the cap, _new_attack_time_counters, _previous_attacks line (-1: None)
AREA_N, AREA_COUNTER, AREA_NEXT, AREA_OVERFLOW, AREA_CLOCK, AREA_PREV = range(6)
MULTI_KEYS = ("multi_mt", "multi_mt_pos", "multi_wait", "multi_dur", "multi_ctr", "multi_fails")   # its keys of get_state()
_COST = np.int64(1)                    # BaseActionBudget of one line's set_line_status action
_INT32_MAX = 2 ** 31 - 1
_LOG_U_MAX = float(np.log(2.0 ** -53))  # log1p(-U) for the largest random_sample(), 1 - 2**-53: the largest geometric draw


def _max_geometric(p: float) -> int:
    """about the largest value ``RandomState.geometric(p)`` can return, ``0 < p <= 1``"""
    return 1 if p >= 1.0 else int(np.ceil(_LOG_U_MAX / np.log1p(-p))) + 1


def geometric_constants(attack_every_xxx_hour, average_attack_duration_hour, minimum_attack_duration_hour, delta_time_seconds=300.0):
    """``GeometricOpponent.init``'s rates: -> (recovery_min int, recovery_rate, attack_hazard_rate); its OpponentError cases and rates
    whose draws would not fit an int32 (grid2op's ``astype(dt_int)`` would wrap them) raise ValueError.  The environment's
    ``delta_time_seconds`` is a float32, so the steps per hour and both rates are float32 values, as in grid2op."""
    ts_per_hour = 3600.0 / np.float32(delta_time_seconds)
    recovery_min = int(minimum_attack_duration_hour * ts_per_hour)
    if average_attack_duration_hour < minimum_attack_duration_hour:
        raise ValueError("The average duration of an attack cannot be lower than the minimum time of an attack")
    if average_attack_duration_hour == minimum_attack_duration_hour:
        raise ValueError("average_attack_duration_hour == minimum_attack_duration_hour is not supported")
    recovery_rate = 1.0 / (ts_per_hour * (average_attack_duration_hour - minimum_attack_duration_hour))
    if attack_every_xxx_hour <= average_attack_duration_hour:
        raise ValueError("attack_every_xxx_hour <= average_attack_duration_hour is not supported")
    hazard_rate = 1.0 / (ts_per_hour * (attack_every_xxx_hour - average_attack_duration_hour))
    for name, p, extra in (("attack hazard", hazard_rate, 0), ("recovery", recovery_rate, recovery_min)):
        if not 0.0 < p <= 1.0:
            raise ValueError(f"the {name} rate {p} is not a probability (fewer than one step per hour?)")
        if recovery_min < 0 or extra + _max_geometric(float(p)) > _INT32_MAX:
            raise ValueError(f"the {name} rate {p} is too small: its draws would not fit an int32")
    return recovery_min, recovery_rate, hazard_rate


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
                 rho_normalization: Optional[Sequence[float]] = None, attack_every_xxx_hour: Optional[float] = None,
                 average_attack_duration_hour: Optional[float] = None, minimum_attack_duration_hour: Optional[float] = None,
                 pmax_pmin_ratio: float = 4, delta_time_seconds: float = 300.0, episode_max_time=None):
        """``GeometricOpponent``: ``attack_every_xxx_hour``, ``average_attack_duration_hour``, ``minimum_attack_duration_hour``,
        ``pmax_pmin_ratio`` (its ``kwargs_opponent``), ``delta_time_seconds`` (the environment's step) and ``episode_max_time`` (int
        or int [batch]: ``env.max_episode_duration()`` of each instance's scenario).  ``GeometricOpponentMultiArea``: the same, with
        ``lines`` a list of areas (lists of line ids)."""
        if kind not in OPPONENT_KINDS:
            raise ValueError(f"unknown opponent {kind!r} ({' / '.join(OPPONENT_KINDS)})")
        self.kind = kind
        self.code = OPPONENT_KINDS[kind]
        self.multi = kind == "GeometricOpponentMultiArea"
        if self.multi:
            areas = [np.asarray(a, dtype=np.int64).reshape(-1) for a in lines]
            if not 1 <= len(areas) <= MAX_AREAS:
                raise ValueError(f"GeometricOpponentMultiArea takes 1 to {MAX_AREAS} areas")
            if any(len(a) == 0 for a in areas):
                raise ValueError("GeometricOpponentMultiArea: an area without lines")
            seen = [set(a.tolist()) for a in areas]
            if any(seen[j] & seen[k] for j in range(len(seen)) for k in range(j)):
                raise ValueError("GeometricOpponentMultiArea: two areas share a line")
            if int(attack_cooldown) >= 2:
                raise ValueError("GeometricOpponentMultiArea needs attack_cooldown 0 or 1: with a longer cooldown OpponentSpace skips "
                                 "a step and grid2op's multi-area tell_attack_continues raises")
            self.area_off = np.concatenate([[0], np.cumsum([len(a) for a in areas])]).astype(np.int32)
            lines = np.concatenate(areas)
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
        self.geometric = kind == "GeometricOpponent"
        if self.geometric or self.multi:
            self._init_geometric(attack_every_xxx_hour, average_attack_duration_hour, minimum_attack_duration_hour, pmax_pmin_ratio,
                                 delta_time_seconds, episode_max_time)
        self.reset(np.arange(batch))

    def _init_geometric(self, every, average, minimum, pmax_pmin_ratio, delta_time_seconds, episode_max_time):
        if every is None or average is None or minimum is None:
            raise ValueError("GeometricOpponent needs attack_every_xxx_hour, average_attack_duration_hour and minimum_attack_duration_hour")
        if not float(pmax_pmin_ratio) > 0.0:
            raise ValueError("pmax_pmin_ratio must be > 0")
        if not float(delta_time_seconds) > 0.0:
            raise ValueError("delta_time_seconds must be > 0")
        self.recovery_min, self.recovery_rate, self.hazard_rate = geometric_constants(every, average, minimum, delta_time_seconds)
        # the divisor of numpy's inversion, log(1 - p) in double precision (RandomState.geometric takes p as a double)
        self.logq_hazard, self.logq_recovery = float(np.log(1.0 - float(self.hazard_rate))), float(np.log(1.0 - float(self.recovery_rate)))
        if episode_max_time is None:
            raise ValueError("GeometricOpponent needs episode_max_time")
        emt = np.broadcast_to(np.asarray(episode_max_time, dtype=np.int64), (self.batch,))
        if (emt < 0).any() or (emt > _INT32_MAX).any():
            raise ValueError("episode_max_time out of range")
        self.emt = emt.astype(np.int32)
        self.pmax_pmin_ratio = pmax_pmin_ratio
        # every appended attack advances the schedule's time by at least recovery_min + 2 (a wait >= 1, a duration >= recovery_min + 1)
        self.cap = int(-(-int(self.emt.max()) // (self.recovery_min + 2))) + 1
        if self.multi:
            self._init_areas()
            return
        n = len(self.lines)
        # GeometricOpponent.attack's expressions, for every rank at once: the lines it weighs are always all attackable lines
        self.b_beta = self._b_beta(n)
        self.geo_weights = np.exp(self.b_beta * np.arange(n, dtype=np.int64))
        self.geo_wait = np.zeros((self.batch, self.cap), dtype=np.int32)
        self.geo_dur = np.zeros((self.batch, self.cap), dtype=np.int32)
        self.geo_ctr = np.zeros((self.batch, 4), dtype=np.int32)         # schedule length, attacks consumed, previous_fails, dropped

    def _b_beta(self, n):
        return np.log(self.pmax_pmin_ratio) / (n - 1) if n > 1 else np.float64(0.0)

    def _init_areas(self):
        """GeometricOpponentMultiArea.init and seed: one GeometricOpponent per area, each seeded from the multi-area opponent's own
        stream (``self.rngs``) in area order"""
        A, B = len(self.area_off) - 1, self.batch
        sizes = np.diff(self.area_off)
        self.area_b_beta = [self._b_beta(int(n)) for n in sizes]
        # each area's weight table at its lines' offsets (the device indexes area_off[k] + rank)
        self.area_weights = np.concatenate([np.exp(b * np.arange(int(n), dtype=np.int64)) for b, n in zip(self.area_b_beta, sizes)])
        max_seed = np.iinfo(np.int32).max
        self.multi_rngs = [[np.random.RandomState(r.randint(max_seed)) for _ in range(A)] for r in self.rngs]
        self.multi_wait = np.zeros((B, A, self.cap), dtype=np.int32)
        self.multi_dur = np.zeros((B, A, self.cap), dtype=np.int32)
        self.multi_ctr = np.zeros((B, A, 6), dtype=np.int32)
        self.multi_ctr[:, :, AREA_CLOCK] = -1
        self.multi_ctr[:, :, AREA_PREV] = -1
        self.area_next = [[None] * A for _ in range(B)]
        self.fails = np.zeros(B, dtype=bool)                             # OpponentSpace.previous_fails

    def _geo_sample(self, rng, emt, wait, dur, ctr):
        """GeometricOpponent.sample_attack_times_and_durations on ``rng``, into one schedule row ``wait`` / ``dur`` [cap] and its
        counters ``ctr`` (schedule length, attacks consumed and entries dropped at the cap in words 0, 1 and 3)"""
        waits, durs = [], []
        t = 0
        while t < emt:
            t_to_attack = rng.geometric(p=self.hazard_rate)
            t = t + t_to_attack
            if t < emt:
                waits.append(t_to_attack)
                d = self.recovery_min + rng.geometric(p=self.recovery_rate)
                durs.append(d)
                t = t + d
        n = min(len(waits), self.cap)
        wait[:n] = np.array(waits[:n]).astype(np.int32)
        dur[:n] = np.array(durs[:n]).astype(np.int32)
        ctr[0], ctr[1] = n, 0
        ctr[3] += len(waits) - n

    # ---- OpponentSpace.reset ----------------------------------------------------------------------------------------------
    def reset(self, idx):
        """the random streams continue"""
        for i in np.asarray(idx, dtype=np.int64).reshape(-1):
            self.budget[i] = self.init_budget
            self.duration[i] = 0
            self.cooldown[i] = int(self.attack_cooldown)
            self.last[i] = -1
            self.next_time[i] = None
            if self.geometric:
                self._geo_sample(self.rngs[i], int(self.emt[i]), self.geo_wait[i], self.geo_dur[i], self.geo_ctr[i])
                self.geo_ctr[i, 2] = 0                                      # previous_fails
            if self.multi:                  # GeometricOpponentMultiArea.reset: every counter to -1, then each area's reset
                self.fails[i] = False
                self.multi_ctr[i, :, AREA_CLOCK] = -1
                for k, rng in enumerate(self.multi_rngs[i]):
                    self._geo_sample(rng, int(self.emt[i]), self.multi_wait[i, k], self.multi_dur[i, k], self.multi_ctr[i, k])
                    self.area_next[i][k] = None

    # ---- OpponentSpace.attack ---------------------------------------------------------------------------------------------
    def attack(self, line_status: np.ndarray, rho: Optional[np.ndarray], live: np.ndarray):
        """One step of every live instance: ``line_status`` bool [B, n_line] and ``rho`` float32 [B, n_line] of the previous step
        (the observation the opponent sees).  -> (attacked line int32 [B], -1 for none; attack duration int32 [B]); a
        GeometricOpponentMultiArea gives the attacked line of every area, int32 [B, n_area] (-1: none in that area)"""
        line = np.full((self.batch, len(self.area_off) - 1) if self.multi else self.batch, -1, dtype=np.int32)
        dur = np.zeros(self.batch, dtype=np.int32)
        one = self._multi_attack_one if self.multi else self._attack_one
        for i in np.flatnonzero(live):
            a, d = one(int(i), line_status[i], None if rho is None else rho[i])
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
            if self.geometric:
                fails = False
                if duration > self.attack_duration:
                    attack, fails = None, True
                if duration * self._cost(attack) > self.budget[i]:
                    attack, fails = None, True
                self.geo_ctr[i, 2] = fails                                  # previous_fails
            elif duration * self._cost(attack) > self.budget[i]:
                attack = None
            if attack is not None:
                self.duration[i] = duration
                self.cooldown[i] += self.attack_cooldown
        if not asked and (self.weighted or self.geometric):
            self.next_time[i] = None                                        # tell_attack_continues
        if not asked and self.geometric:
            self.geo_ctr[i, 2] = 0
        self.budget[i] = self.budget[i] - self._cost(attack)
        self.last[i] = -1 if attack is None else attack
        return (-1, 0) if attack is None else (attack, int(self.duration[i]))

    @staticmethod
    def _cost(attack):
        return 0 if attack is None else _COST

    @staticmethod
    def _geo_attack(rng, wait, dur, ctr, next_time, fails, lines, b_beta, status, rho):
        """GeometricOpponent.attack of one opponent: its stream, schedule row and counters (as :meth:`_geo_sample` writes them), its
        ``_next_attack_time``, OpponentSpace's ``previous_fails``, its lines and ``b_beta`` -> (line or None, duration or None,
        ``_next_attack_time``)"""
        n, c = int(ctr[0]), int(ctr[1])
        if c >= n:
            return None, None, next_time
        wait, dur = wait[:n], dur[:n]
        if fails:
            next_time = wait[c] + dur[c - 1]
        if next_time is None:
            next_time = 1 + wait[c]
        attack_duration = dur[c]
        next_time -= 1
        if next_time > 0:
            return None, None, next_time
        ctr[1] = c + 1
        st = np.asarray(status, dtype=bool)[lines]
        if ~st.all():
            return None, None, next_time
        if len(lines) == 1:
            return int(lines[0]), attack_duration, next_time
        r = np.asarray(rho, dtype=np.float32)[lines]
        temp = r.argsort(kind="stable")
        rho_ranks = np.empty_like(temp)
        rho_ranks[temp] = np.arange(len(r))
        raw_probabilities = np.exp(b_beta * rho_ranks)
        b_probabilities = raw_probabilities / raw_probabilities.sum()
        return int(rng.choice(lines, p=b_probabilities)), attack_duration, next_time

    def _multi_attack_one(self, i, status, rho):
        """OpponentSpace.attack with GeometricOpponentMultiArea.attack -> (line int32 [n_area], -1 where none; duration)"""
        self.budget[i] = self.budget[i] + self.budget_per_ts
        self.duration[i] = max(0, self.duration[i] - 1)
        self.cooldown[i] = max(0, self.cooldown[i] - 1)
        if self.duration[i] > 0 or self.cooldown[i] > self.attack_cooldown:     # (attack_cooldown <= 1 and duration 1: never)
            raise RuntimeError("OpponentSpace skipped the GeometricOpponentMultiArea, whose tell_attack_continues raises")
        ctr = self.multi_ctr[i]
        ctr[:, AREA_CLOCK] -= 1
        ctr[ctr[:, AREA_CLOCK] < -1, AREA_CLOCK] = -1
        fails = self.fails[i]
        for k in range(len(ctr)):
            if ctr[k, AREA_CLOCK] == -1:
                lines = self.lines[self.area_off[k]:self.area_off[k + 1]]
                a, d, self.area_next[i][k] = self._geo_attack(self.multi_rngs[i][k], self.multi_wait[i, k], self.multi_dur[i, k], ctr[k],
                                                              self.area_next[i][k], fails, lines, self.area_b_beta[k], status, rho)
                if a is not None:
                    ctr[k, AREA_CLOCK] = d
                ctr[k, AREA_PREV] = -1 if a is None else a
            else:
                self.area_next[i][k] = None                                 # tell_attack_continues
        out = ctr[:, AREA_PREV].astype(np.int32)                            # the combined attack: every area's remembered line
        n = int((out >= 0).sum())
        attack, duration, fails = n > 0, 1, False
        if duration > self.attack_duration:
            attack, fails = False, True
        if duration * (np.int64(n) if attack else 0) > self.budget[i]:
            attack, fails = False, True
        self.fails[i] = fails
        if attack:
            self.duration[i] = duration
            self.cooldown[i] += self.attack_cooldown
        else:
            out[:] = -1
        self.budget[i] = self.budget[i] - (np.int64(n) if attack else 0)
        self.last[i] = out[out >= 0][0] if attack else -1
        return out, (int(self.duration[i]) if attack else 0)

    def _opponent_attack(self, i, status, rho):
        rng = self.rngs[i]
        if self.geometric:
            a, d, self.next_time[i] = self._geo_attack(rng, self.geo_wait[i], self.geo_dur[i], self.geo_ctr[i], self.next_time[i],
                                                       self.geo_ctr[i, 2], self.lines, self.b_beta, status, rho)
            return a, d
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
        """-> dict(budget float64 [B], budget64 uint8 [B], ctr int32 [B, 4], mt uint32 [B, 624], mt_pos int32 [B]); a
        GeometricOpponent adds geo_wait / geo_dur int32 [B, cap] (the schedules) and geo_ctr int32 [B, 4] (schedule length, attacks
        consumed, previous_fails, schedule entries dropped at the cap); a GeometricOpponentMultiArea adds its areas' streams
        multi_mt uint32 [B, n_area, 624] / multi_mt_pos int32 [B, n_area], their schedules multi_wait / multi_dur int32
        [B, n_area, cap], their counters multi_ctr int32 [B, n_area, 6] (schedule length, attacks consumed, _next_attack_time,
        entries dropped at the cap, _new_attack_time_counters, _previous_attacks line) and multi_fails int32 [B] (previous_fails);
        its mt / mt_pos are the multi-area opponent's own stream, which only seeded the areas"""
        B = self.batch
        ctr = np.empty((B, 4), dtype=np.int32)
        ctr[:, 0], ctr[:, 1], ctr[:, 2] = self.duration, self.cooldown, self.last
        ctr[:, 3] = [NEXT_UNSET if t is None else int(t) for t in self.next_time]
        mt = np.empty((B, 624), dtype=np.uint32)
        pos = np.empty(B, dtype=np.int32)
        for i, r in enumerate(self.rngs):
            st = r.get_state()
            mt[i], pos[i] = st[1], st[2]
        s = dict(budget=np.array([float(b) for b in self.budget], dtype=np.float64),
                 budget64=np.array([b.dtype == np.float64 for b in self.budget], dtype=np.uint8), ctr=ctr, mt=mt, mt_pos=pos)
        if self.geometric:
            s.update(geo_wait=self.geo_wait.copy(), geo_dur=self.geo_dur.copy(), geo_ctr=self.geo_ctr.copy())
        if self.multi:
            A = len(self.area_off) - 1
            amt = np.empty((B, A, 624), dtype=np.uint32)
            apos = np.empty((B, A), dtype=np.int32)
            for i in range(B):
                for k, r in enumerate(self.multi_rngs[i]):
                    st = r.get_state()
                    amt[i, k], apos[i, k] = st[1], st[2]
            actr = self.multi_ctr.copy()
            actr[:, :, AREA_NEXT] = [[NEXT_UNSET if t is None else int(t) for t in row] for row in self.area_next]
            s.update(multi_mt=amt, multi_mt_pos=apos, multi_wait=self.multi_wait.copy(), multi_dur=self.multi_dur.copy(),
                     multi_ctr=actr, multi_fails=self.fails.astype(np.int32))
        return s

    def set_state(self, s):
        for i in range(self.batch):
            self.budget[i] = np.float64(s["budget"][i]) if s["budget64"][i] else np.float32(s["budget"][i])
            self.rngs[i].set_state(("MT19937", np.asarray(s["mt"][i], dtype=np.uint32), int(s["mt_pos"][i]), 0, 0.0))
        self.duration[:], self.cooldown[:], self.last[:] = s["ctr"][:, 0], s["ctr"][:, 1], s["ctr"][:, 2]
        if self.geometric:              # (grid2op keeps _next_attack_time as a numpy int32)
            self.next_time = [None if int(t) == NEXT_UNSET else np.int32(t) for t in s["ctr"][:, 3]]
            self.geo_wait[:], self.geo_dur[:], self.geo_ctr[:] = s["geo_wait"], s["geo_dur"], s["geo_ctr"]
        else:
            self.next_time = [None if int(t) == NEXT_UNSET else int(t) for t in s["ctr"][:, 3]]
        if self.multi:
            for i in range(self.batch):
                for k, r in enumerate(self.multi_rngs[i]):
                    r.set_state(("MT19937", np.asarray(s["multi_mt"][i, k], dtype=np.uint32), int(s["multi_mt_pos"][i, k]), 0, 0.0))
            self.multi_wait[:], self.multi_dur[:], self.multi_ctr[:] = s["multi_wait"], s["multi_dur"], s["multi_ctr"]
            self.area_next = [[None if int(t) == NEXT_UNSET else np.int32(t) for t in row] for row in s["multi_ctr"][:, :, AREA_NEXT]]
            self.fails[:] = np.asarray(s["multi_fails"]) != 0
