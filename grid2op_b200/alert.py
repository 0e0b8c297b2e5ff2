"""grid2op's line alerts (l2rpn_idf_2023) for a whole batch, on the host: the environment's alert state and the AlertReward.

Reference (grid2op 1.12.5), per environment:

* ``BaseEnv._update_alert_properties`` (grid2op/Environment/baseEnv.py:3295-3335): run after the opponent's attack, before the
  power flow; ``lines_attacked`` is the attack's topological impact (every step of an ongoing attack), ``None`` without an attack;
* ``BaseEnv._reset_alert`` (baseEnv.py:1677-1685) at ``env.reset()``;
* ``AlertReward`` (grid2op/Reward/alertReward.py): a ring of ``ALERT_TIME_WINDOW + 2`` rows of "newly attacked" and "alert
  launched" flags; it writes ``env._was_alert_used_after_attack``, which the observation copies in ``update_after_reward``.

:class:`BatchedAlerts` keeps the same arrays as the device (csrc/b200pf_alert.cuh, ``b200pf_alert_get_state``) so that the two
paths hand the state over as it is.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np

__all__ = ["BatchedAlerts", "ALERT_STATE"]

# the state arrays in the order of b200pf_alert_get_state / _set_state
ALERT_STATE = (("last_alert", np.uint8), ("already", np.uint8), ("tsl_alert", np.int32), ("duration", np.int32),
               ("tsl_attack", np.int32), ("under_alert", np.int32), ("was_used", np.int32), ("total", np.int32),
               ("ts_attack", np.uint8), ("launched", np.uint8), ("current", np.uint8), ("cur_id", np.int32))


class BatchedAlerts:
    def __init__(self, lines, batch: int, *, window: int = 12, reward: bool = True, reward_min_no_blackout=-1.0,
                 reward_min_blackout=-10.0, reward_max_no_blackout=1.0, reward_max_blackout=2.0, reward_end_episode_bonus=1.0):
        self.lines = np.asarray(lines, dtype=np.int32)
        self.n, self.batch, self.window, self.ring, self.reward = len(self.lines), int(batch), int(window), int(window) + 2, bool(reward)
        f = np.float32
        # AlertReward.__init__: float32 constants, the two differences taken in float32
        self.min_blackout = f(reward_min_blackout)
        self.range_blackout = f(reward_max_blackout) - f(reward_min_blackout)
        self.max_no_blackout = f(reward_max_no_blackout)
        self.diff_no_blackout = f(reward_min_no_blackout) - f(reward_max_no_blackout)
        self.constants = dict(reward_min_no_blackout=f(reward_min_no_blackout), reward_min_blackout=f(reward_min_blackout),
                              reward_max_no_blackout=f(reward_max_no_blackout), reward_max_blackout=f(reward_max_blackout),
                              reward_end_episode_bonus=f(reward_end_episode_bonus))
        B, n, R = self.batch, self.n, self.ring
        self.s: Dict[str, np.ndarray] = {}
        for k, dt in ALERT_STATE:
            shape = (B,) if k in ("total", "cur_id") else (B, R, n) if k in ("ts_attack", "launched") else (B, n)
            self.s[k] = np.zeros(shape, dtype=dt)
        self.reward_out = np.zeros(B, dtype=np.float64)
        self.reset(np.arange(B))

    def reset(self, idx):
        """``_reset_alert`` + ``AlertReward.reset`` of the instances ``idx``"""
        s = self.s
        for k in s:
            s[k][idx] = 0
        s["tsl_alert"][idx] = -1
        s["tsl_attack"][idx] = -1
        self.reward_out[idx] = 0.0

    def _attacked(self, attack: Optional[np.ndarray]):
        """-> (hit bool [B, n]: alertable line attacked this step, any bool [B]: the step has an attack)"""
        B = self.batch
        if attack is None:
            return np.zeros((B, self.n), bool), np.zeros(B, bool)
        at = np.asarray(attack).reshape(B, -1)
        hit = (at[:, :, None] == self.lines[None, None, :]).any(axis=1)
        return hit, (at >= 0).any(axis=1)

    def step(self, raise_alert: Optional[np.ndarray], attack: Optional[np.ndarray], live: np.ndarray, blackout: np.ndarray):
        """one ordinary step: ``raise_alert`` bool [B, n] (None: no alert), ``attack`` the opponent's lines of the step (int [B] or
        [B, n_area], -1: none; None: no opponent), ``live`` bool [B] (not finished before the step), ``blackout`` bool [B] (the step
        ended the episode).  Updates the state of the live instances and the reward of every instance (0 for the others)."""
        s, B, n = self.s, self.batch, self.n
        up = np.zeros((B, n), bool) if raise_alert is None else np.asarray(raise_alert, dtype=bool).reshape(B, n)
        hit, any_att = self._attacked(attack)
        L = np.asarray(live, dtype=bool)
        Lk = np.repeat(L[:, None], n, axis=1)
        # _update_alert_properties
        s["last_alert"][L] = up[L]
        t = s["tsl_alert"]
        t[Lk & ~up & (t != -1)] += 1
        t[Lk & up] = 0
        d = s["duration"]
        d[Lk & up] += 1
        d[Lk & ~up] = 0
        s["total"][L] += up[L].sum(axis=1).astype(np.int32)
        ta, al = s["tsl_attack"], s["already"]
        A = (Lk & any_att[:, None])
        first = A & hit & (al == 0)
        ta[first] = 0
        ta[A & ~first & (ta != -1)] += 1
        al[A & hit] = 1
        N = Lk & ~any_att[:, None]
        ta[N & (ta != -1)] += 1
        al[N] = 0
        ua = s["under_alert"]
        new = Lk & (ta == 0)
        ua[new] = np.where(up[new], 1, -1)
        ua[Lk & (ta > self.window)] = 0
        self.reward_out[:] = 0.0
        if self.reward:
            for i in np.flatnonzero(L):
                self.reward_out[i] = self._reward_instance(i, up[i], hit[i], bool(any_att[i]), bool(blackout[i]))
        return self.reward_out

    def _reward_instance(self, i, up, hit, any_att, blackout):
        """AlertReward._update_state + __call__ of instance i"""
        s, R, W = self.s, self.ring, self.window
        ts, la, cur, used = s["ts_attack"][i], s["launched"][i], s["current"][i], s["was_used"][i]
        cid = (int(s["cur_id"][i]) + 1) % R
        s["cur_id"][i] = cid
        if not any_att:
            cur[:] = 0
            ts[cid, :] = 0
        else:
            ts[cid, hit & (cur == 0)] = 1
            cur[:] = hit
        la[cid, :] = up
        used[:] = 0
        if blackout:
            rows = (np.arange(-W, 1) + cid) % R
            win = ts[rows].astype(bool)
            if not win.any():
                return 0.0
            ti, li = win.nonzero()
            line_first, first_idx = np.unique(li, return_index=True)
            prev = rows[ti[first_idx]]
            sent = la[prev, line_first].astype(bool)
            used[line_first] = np.where(sent, 1, -1)
            return float(np.mean(sent) * self.range_blackout + self.min_blackout)
        r = (cid - W) % R
        att = ts[r].astype(bool)
        if not att.any():
            return 0.0
        sent = la[r, att].astype(bool)
        used[att] = np.where(sent, -1, 1)
        ts[r, :] = 0
        return float(self.diff_no_blackout * np.mean(sent) + self.max_no_blackout)

    def obs_record(self) -> np.ndarray:
        """int32 [B, 6 n + 1]: the alert values of the observe input record (alert_obs_record of csrc/b200pf_alert.cuh)"""
        s = self.s
        return np.concatenate([s["last_alert"], s["under_alert"], s["tsl_alert"], s["duration"], s["total"][:, None], s["tsl_attack"],
                               s["was_used"]], axis=1).astype(np.int32)

    def get_state(self) -> Dict[str, np.ndarray]:
        return {k: v.copy() for k, v in self.s.items()}

    def set_state(self, st: Dict[str, np.ndarray]):
        for k, dt in ALERT_STATE:
            self.s[k][:] = np.asarray(st[k], dtype=dt).reshape(self.s[k].shape)
