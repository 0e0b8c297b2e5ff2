"""Batched ``env.step`` WITH actions: the driver next to :class:`grid2op_b200.rollout.BatchedDoNothing` for agents that
act on the topology (BASELINE.json configs[2]: "random topology actions"), with the environment-side bookkeeping a
topology agent depends on.

What one :meth:`BatchedEnv.step` restates for a whole batch of independent environments (reference, per env —
``BaseEnv.step`` grid2op/Environment/baseEnv.py:3778-3872 and what it calls), for the action subset
{do nothing, set the busbars of ONE substation, set the status of ONE line} (the ``sub_id`` / ``line_id`` arguments), or
grid2op's native topology action (``set_bus`` / ``change_bus`` / ``set_line_status`` / ``change_line_status`` vectors,
:meth:`BatchedEnv._apply_actions`):

1. legality — ``LookParam`` (``max_sub_changed`` / ``max_line_status_changed``, grid2op/Parameters.py:279; or the same maxima per
   area of ``RulesByArea``) and ``PreventReconnection``: an action that touches a line whose ``times_before_line_status_actionable``
   is > 0 or a substation whose ``times_before_topology_actionable`` is > 0 is illegal and replaced by "do nothing"
   (grid2op/Rules/PreventReconnection.py:33-60, baseEnv.py:3798-3820);
2. ``_backend_action += action`` (baseEnv.py:3822-3846): busbars of the substation's elements, line disconnection
   (both ends -1) / reconnection (each end back on its last busbar, grid2op/Action/_backendAction.py ``last_topo_registered``);
   a busbar > 0 for the end of a DISCONNECTED line inside a substation action reconnects that line (the line, not the
   substation, is what such an entry impacts: grid2op/Action/baseAction.py:1836-1860);
3. the environment's own modifications of this step: next chronics row (gridStateFromFile.py:766-776), lines in
   ``maintenance`` / ``hazards`` forced out (gridStateFromFile.py:780-797, baseAction ``maintenance`` / ``hazards`` keys);
4. ``backend.next_grid_state`` — one batched power flow with the protections of backend.py:1433-1521 on the device;
5. the cooldown bookkeeping of baseEnv.py:3352-3393: line cooldowns decrease, lines tripped by the protections get
   ``NB_TIMESTEP_RECONNECTION``, maintenance / hazard durations are folded in (baseEnv.py:2566-2597), lines / substations
   the (legal) action named get ``NB_TIMESTEP_COOLDOWN_LINE`` / ``NB_TIMESTEP_COOLDOWN_SUB``;
6. game over when the power flow fails (baseEnv.py:3523-3524); a finished instance stays finished.

The topology lives on the HOST (int8 [batch, n_topo_in]); a step that changed it hands the rows to
``PowerFlowEngine.series_set_topo`` — cached plans are looked up by hash, new topologies are planned on the host threads
(see DESIGN.md "config 3").  Everything numeric stays on the device as in :class:`BatchedDoNothing`.
"""
from __future__ import annotations

import os
from typing import Optional

import numpy as np

from .gridmodel import GridModel
from .rollout import BatchedDoNothing

__all__ = ["BatchedEnv", "random_substation_actions"]


class BatchedEnv(BatchedDoNothing):
    def __init__(self, gm: GridModel, chron: np.ndarray, batch: int, *, maintenance: Optional[np.ndarray] = None,
                 hazards: Optional[np.ndarray] = None, nb_timestep_cooldown_line: int = 0, nb_timestep_cooldown_sub: int = 0,
                 nb_timestep_reconnection: int = 10, engine=None, tight_cap: bool = True, max_sub_changed: int = 1,
                 max_line_status_changed: int = 1, rules_by_area=None, **kw):
        """``maintenance`` / ``hazards``: bool [n_scen, n_rows, n_line] (:func:`grid2op_b200.chronics.load_line_events` per
        scenario), row-aligned with ``chron``.  Cooldown parameters: grid2op.Parameters NB_TIMESTEP_COOLDOWN_LINE /
        NB_TIMESTEP_COOLDOWN_SUB / NB_TIMESTEP_RECONNECTION (Parameters.py:255-300).  Legality: ``max_sub_changed`` /
        ``max_line_status_changed`` are MAX_SUB_CHANGED / MAX_LINE_STATUS_CHANGED; ``rules_by_area``, a list of lists of substation
        ids as ``RulesByArea(areas_list)`` takes them, applies these maxima per area instead of over the whole grid (at most 16
        areas).  Without it the rules are ``LookParam`` + ``PreventReconnection`` (``DefaultRules`` at the default maxima)."""
        if int(max_sub_changed) < 0 or int(max_line_status_changed) < 0:
            raise ValueError("max_sub_changed and max_line_status_changed must be >= 0")
        super().__init__(gm, chron, batch, engine=engine, **kw)
        B, nl = self.batch, gm.n_line
        self.topo = self.topo0.copy()                                      # int8 [B, n_topo_in], -1 = disconnected
        self.last_bus = np.where(self.topo[:, :gm.dim_topo] > 0, self.topo[:, :gm.dim_topo], 1).astype(np.int8)
        self.line_cooldown = np.zeros((B, nl), dtype=np.int32)             # times_before_line_status_actionable
        self.sub_cooldown = np.zeros((B, gm.n_sub), dtype=np.int32)        # times_before_topology_actionable
        self.done = np.zeros(B, dtype=bool)
        self.row = self.t0.astype(np.int64).copy()                         # chronics row the NEXT solve uses
        self.cd_line, self.cd_sub, self.cd_reco = int(nb_timestep_cooldown_line), int(nb_timestep_cooldown_sub), int(nb_timestep_reconnection)
        self._maint = self._maint_time = self._maint_dur = self._haz = self._haz_dur = None
        if maintenance is not None:
            from .chronics import maintenance_time_duration
            self._maint = np.asarray(maintenance, dtype=bool)
            td = [maintenance_time_duration(m) for m in self._maint]
            self._maint_time = np.stack([x[0] for x in td]); self._maint_dur = np.stack([x[1] for x in td])
        if hazards is not None:
            from .chronics import hazard_duration
            self._haz = np.asarray(hazards, dtype=bool)
            self._haz_dur = np.stack([hazard_duration(h) for h in self._haz])
        # element positions of every substation in the topology vector (grid2op order), padded
        sub_of = np.full(gm.dim_topo, -1, dtype=np.int64)
        sub_of[gm.line_or_pos] = gm.line_or_sub; sub_of[gm.line_ex_pos] = gm.line_ex_sub
        sub_of[gm.gen_pos] = gm.gen_sub; sub_of[gm.load_pos] = gm.load_sub
        if gm.n_storage:
            sub_of[gm.storage_pos] = gm.storage_sub
        self.sub_of_pos = sub_of
        self.sub_size = np.bincount(sub_of, minlength=gm.n_sub)
        self.max_sub_size = int(self.sub_size.max())
        self.sub_pos = np.full((gm.n_sub, self.max_sub_size), -1, dtype=np.int64)
        for s in range(gm.n_sub):
            p = np.flatnonzero(sub_of == s)
            self.sub_pos[s, :len(p)] = p
        self.line_or_pos, self.line_ex_pos = np.asarray(gm.line_or_pos, dtype=np.int64), np.asarray(gm.line_ex_pos, dtype=np.int64)
        # line whose end sits at a position of the topology vector (-1: not a line end) and the position of its other end
        self.line_of_pos = np.full(gm.dim_topo, -1, dtype=np.int64)
        self.other_end_pos = np.full(gm.dim_topo, -1, dtype=np.int64)
        self.line_of_pos[self.line_or_pos] = np.arange(nl); self.line_of_pos[self.line_ex_pos] = np.arange(nl)
        self.other_end_pos[self.line_or_pos] = self.line_ex_pos; self.other_end_pos[self.line_ex_pos] = self.line_or_pos
        self._topo_dirty = False
        self.max_sub_changed, self.max_line_status_changed = int(max_sub_changed), int(max_line_status_changed)
        self._set_rules_by_area(rules_by_area)
        self._pos_sub = np.zeros((gm.dim_topo, gm.n_sub), dtype=np.int64)             # one-hot substation of each position
        self._pos_sub[np.arange(gm.dim_topo), sub_of] = 1
        # Shunts: this driver never acts on them, so the environment of the reference holds every shunt for connected to busbar 1
        # (_BackendAction.current_shunt_bus, grid2op/Action/_backendAction.py:513-514) and counts that busbar as active
        # (:1519-1531 -> bus.in_service, pandaPowerBackend.py:920-922) — also when the grid file has the shunt out of service (all six of
        # l2rpn_neurips_2020_track1).  Busbar 1 of such a substation must keep an element: :meth:`_isolated_shunt_busbar`.
        self._shunt_off = np.flatnonzero(self.topo0[0, gm.dim_topo:gm.dim_topo + gm.n_shunt] <= 0) if gm.n_shunt else np.zeros(0, dtype=np.int64)
        self._shunt_off_pos = [self.sub_pos[int(gm.shunt_sub[k]), :self.sub_size[int(gm.shunt_sub[k])]] for k in self._shunt_off]
        hid_sub = np.asarray(gm.hidden_sub, dtype=np.int64) if gm.n_hidden else np.zeros(0, dtype=np.int64)
        on_sub = np.asarray(gm.shunt_sub, dtype=np.int64)[np.setdiff1d(np.arange(gm.n_shunt), self._shunt_off)] if gm.n_shunt else hid_sub
        self._iso_cols = self._iso_seg = None
        self._shunt_off_other = [bool(np.isin(int(gm.shunt_sub[k]), hid_sub) or np.isin(int(gm.shunt_sub[k]), on_sub)) for k in self._shunt_off]
        # Bus splits add active buses: the kernels that discover the topology on the device size their workspace (and the
        # threads per instance) for ``nb_cap`` active buses.  The host knows every instance's topology, so the cap is the
        # bus count of the fullest instance (:meth:`_bus_cap`: host code of the library, recomputed when a topology changed) instead of every bus slot.
        self.tight_cap = bool(tight_cap)
        self._nb_inst = np.zeros(B, dtype=np.int32)                        # active buses per instance (kept incrementally)
        self._cap_dirty = np.ones(B, dtype=bool)                           # instances whose topology changed since it was counted
        self.nb_cap = self._bus_cap() if self.tight_cap else 0
        self.n_illegal = 0
        self.n_steps = 0
        self.is_illegal = np.zeros(B, dtype=bool)                          # the last step's action was replaced by "do nothing"
        self.is_ambiguous = np.zeros(B, dtype=bool)                        # ... as ambiguous (the vector action)
        self.current_step = np.zeros(B, dtype=np.int32)                    # env.nb_time_step (obs.current_step)
        self.soft_overflow_threshold = float(kw.get("soft_overflow_threshold", 1.0))
        self._obs = None
        # tensor path (:meth:`step_tensors`): device buffers of the per-instance state, and where that state lives now ("host" or
        # "device"); a host-path call pulls it, the next step_tensors pushes it back
        self._dev = None
        self._authority = "host"
        self._opp = None                                                   # line-attack opponent (:meth:`enable_opponent`)
        self._alerts = None                                                # line alerts (:meth:`enable_alerts`)
        self._alarms = None                                                # alarms (:meth:`enable_alarms`)
        self._table = None                                                 # discrete action table (:meth:`set_action_table`)

    # ------------------------------------------------------------------------------------------------------------
    def _set_rules_by_area(self, areas):
        """``RulesByArea.__init__`` + ``initialize`` (grid2op/Rules/rulesByArea.py): each area's substations sorted and de-duplicated,
        as many listed as the grid has (ValueError where grid2op raises Grid2OpException), a line in the area of its origin
        substation.  -> ``self.areas`` (None or the areas' substation ids), ``self.lines_id_by_area``, the area masks ``_sub_area`` /
        ``_line_area`` (uint32, bit k: area k) and the membership matrices the counts use (one area of everything without areas)."""
        gm = self.gm
        self.areas = self.lines_id_by_area = self._sub_area = self._line_area = None
        if areas is None:
            self._sub_area_mat = np.ones((gm.n_sub, 1), dtype=np.int64)
            self._line_area_mat = np.ones((gm.n_line, 1), dtype=np.int64)
            return
        areas = [np.unique(np.asarray(list(a), dtype=np.int64)) for a in areas]
        if not 1 <= len(areas) <= 16:
            raise ValueError(f"{len(areas)} areas, 1 to 16 supported")
        if sum(len(a) for a in areas) != gm.n_sub:
            raise ValueError(f"the areas list {sum(len(a) for a in areas)} substations, the grid has {gm.n_sub}")
        if any(((a < 0) | (a >= gm.n_sub)).any() for a in areas):
            raise ValueError("substation id out of range in rules_by_area")
        line_or_sub = np.asarray(gm.line_or_sub, dtype=np.int64)
        self.areas = areas
        self.lines_id_by_area = [np.flatnonzero(np.isin(line_or_sub, a)) for a in areas]
        self._sub_area_mat = np.zeros((gm.n_sub, len(areas)), dtype=np.int64)
        self._line_area_mat = np.zeros((gm.n_line, len(areas)), dtype=np.int64)
        for k, (a, l) in enumerate(zip(areas, self.lines_id_by_area)):
            self._sub_area_mat[a, k] = 1
            self._line_area_mat[l, k] = 1
        w = np.left_shift(np.uint32(1), np.arange(len(areas), dtype=np.uint32))
        self._sub_area = (self._sub_area_mat.astype(np.uint32) * w).sum(axis=1).astype(np.uint32)
        self._line_area = (self._line_area_mat.astype(np.uint32) * w).sum(axis=1).astype(np.uint32)

    def _illegal(self, aff_l, aff_s) -> np.ndarray:
        """bool [B]: the legality rules on an action's topological impact, ``aff_l`` [B, n_line] / ``aff_s`` [B, n_sub] (counts or
        bools): LookParam's maxima over the whole grid or RulesByArea._lookparam_byarea's per area, and PreventReconnection (an
        impacted line or substation in cooldown), grid2op/Rules/LookParam.py, rulesByArea.py, PreventReconnection.py:33-60"""
        aff_l, aff_s = np.asarray(aff_l, dtype=np.int64), np.asarray(aff_s, dtype=np.int64)
        bad = ((aff_l @ self._line_area_mat) > self.max_line_status_changed).any(axis=1)
        bad |= ((aff_s @ self._sub_area_mat) > self.max_sub_changed).any(axis=1)
        bad |= ((aff_l > 0) & (self.line_cooldown > 0)).any(axis=1) | ((aff_s > 0) & (self.sub_cooldown > 0)).any(axis=1)
        return bad

    def _bus_cap(self) -> int:
        """Active buses (bus slots with a connected element) of the fullest instance, rounded up to a multiple of 8 above 17
        (<= 17: exact — the warp-per-instance kernel takes systems up to 17 buses), at most every bus slot.  Per-instance counts are
        kept; only the instances whose topology changed since the last call are counted again (lines tripped by the protections
        only remove buses: the kept count stays an upper bound)."""
        rows = np.flatnonzero(self._cap_dirty)
        if len(rows) == self.batch:
            self._nb_inst[:] = self.engine.max_active_buses(self.topo, per_instance=True)[1]
        elif len(rows):                   # only the instances whose topology changed are counted again
            self._nb_inst[rows] = self.engine.max_active_buses(self.topo[rows], per_instance=True)[1]
        self._cap_dirty[:] = False
        n = int(self._nb_inst.max())
        if n > 17:
            n = (n + 7) // 8 * 8
        return min(n, self.gm.n_slot)

    def line_status(self) -> np.ndarray:
        self._to_host()
        return (self.topo[:, self.line_or_pos] > 0) & (self.topo[:, self.line_ex_pos] > 0)

    def _apply_agent(self, sub_id, sub_bus, line_id, line_status):
        """-> (aff_lines bool [B, n_line], aff_subs bool [B, n_sub]) of the LEGAL actions, applied to self.topo"""
        self._to_host()
        gm, B = self.gm, self.batch
        aff_l = np.zeros((B, gm.n_line), dtype=bool)
        aff_s = np.zeros((B, gm.n_sub), dtype=bool)
        has_sub = np.zeros(B, dtype=bool)
        has_line = np.zeros(B, dtype=bool)
        if sub_id is not None:
            sub_id = np.asarray(sub_id, dtype=np.int64)
            sub_bus = np.asarray(sub_bus, dtype=np.int8)
            has_sub = (sub_id >= 0) & (np.abs(sub_bus) > 0).any(axis=1)
        if line_id is not None:
            line_id = np.asarray(line_id, dtype=np.int64)
            line_status = np.asarray(line_status, dtype=np.int64)
            has_line = (line_id >= 0) & (line_status != 0)
        # A busbar > 0 for the end of a DISCONNECTED line is a reconnection of that line (reference: BaseAction.get_topological_impact,
        # grid2op/Action/baseAction.py:1836-1860 — the line counts as impacted, its two ends do not count for the substation; applied by
        # _BackendAction: the other end goes back to its last busbar)
        reco = None
        sub_impacted = has_sub.copy()
        cnt_l = np.zeros((B, gm.n_line), dtype=np.int64)  # impacted lines (each reconnecting entry counts once) and substations
        cnt_s = np.zeros((B, gm.n_sub), dtype=np.int64)
        reco_is_line = np.zeros(B, dtype=bool)           # the explicitly named line is one of the reconnected ones
        if has_sub.any():
            who_s = np.flatnonzero(has_sub)
            pos = self.sub_pos[sub_id[who_s]]                                    # [n, max_sub_size]
            val = sub_bus[who_s][:, :self.max_sub_size]
            m = (pos >= 0) & (val > 0)
            psafe = np.where(pos >= 0, pos, 0)
            assert self.topo.flags.c_contiguous and self.last_bus.flags.c_contiguous
            tflat, lflat = self.topo.reshape(-1), self.last_bus.reshape(-1)       # (views: both arrays are C-contiguous)
            ft = who_s[:, None] * self.topo.shape[1] + psafe                      # flat indices of the named entries
            cur = tflat[ft]
            dead = m & (cur <= 0)
            if dead.any():                                                        # rare: some named element is disconnected
                lp = np.where(pos >= 0, self.line_of_pos[psafe], -1)
                reco = dead & (lp >= 0)
                if reco.any():
                    np.add.at(cnt_l, (np.broadcast_to(who_s[:, None], pos.shape)[reco], lp[reco]), 1)
                    if line_id is not None:
                        reco_is_line[who_s] = (reco & (lp == np.where(has_line[who_s], line_id[who_s], -2)[:, None])).any(axis=1)
                    sub_impacted[who_s] = (m & ~reco).any(axis=1)
                else:
                    reco = None
        # legality (:meth:`_illegal`) on what the action impacts; finished instances ignore their action
        if sub_id is not None:
            w = np.flatnonzero(has_sub & sub_impacted)
            cnt_s[w, sub_id[w]] = 1
        if line_id is not None:
            w = np.flatnonzero(has_line & ~reco_is_line)
            cnt_l[w, line_id[w]] += 1
        illegal = self._illegal(cnt_l, cnt_s)
        self.n_illegal += int((illegal & ~self.done).sum())
        self.is_illegal = illegal & ~self.done
        ok = ~illegal & ~self.done
        if has_sub.any():
            keep = ok[who_s]
            if keep.any():
                sel = m & (cur > 0) & keep[:, None]                                # connected elements of the legal actions
                fl = who_s[:, None] * self.last_bus.shape[1] + psafe
                tflat[ft[sel]] = val[sel]
                lflat[fl[sel]] = val[sel]
                if reco is not None:                                              # reconnections: this end on the named busbar, the other on its last one
                    rk = reco & keep[:, None]
                    if rk.any():
                        ir = np.broadcast_to(who_s[:, None], pos.shape)[rk]
                        pr, vr = pos[rk], val[rk]
                        po = self.other_end_pos[pr]
                        self.topo[ir, pr] = vr; self.last_bus[ir, pr] = vr
                        self.topo[ir, po] = self.last_bus[ir, po]
                        aff_l[ir, self.line_of_pos[pr]] = True
                who = who_s[keep & sub_impacted[who_s]]
                aff_s[who, sub_id[who]] = True
                self._topo_dirty = True
                self._cap_dirty[who_s[keep]] = True
        if has_line.any():
            who = np.flatnonzero(has_line & ok)
            if len(who):
                l = line_id[who]
                po, pe = self.line_or_pos[l], self.line_ex_pos[l]
                off = line_status[who] < 0
                self.topo[who[off], po[off]] = -1; self.topo[who[off], pe[off]] = -1
                on = ~off
                self.topo[who[on], po[on]] = self.last_bus[who[on], po[on]]
                self.topo[who[on], pe[on]] = self.last_bus[who[on], pe[on]]
                aff_l[who, l] = True
                self._topo_dirty = True
                self._cap_dirty[who] = True
        return aff_l, aff_s

    def _apply_actions(self, sb, cb, ss, cs):
        """grid2op's native topology action (``set_bus`` int [B, dim_topo], ``change_bus`` bool [B, dim_topo], ``set_line_status`` int
        [B, n_line], ``change_line_status`` bool [B, n_line], checked by :meth:`_vector_action`) in BaseEnv.step's order
        (baseEnv.py:3706-3767): BaseAction's topology ambiguity (baseAction.py:3558-3565, :3670-3771), the topological impact on the
        line status the previous step left (:1796-2022), legality (:meth:`_illegal`), and _BackendAction.__iadd__'s application
        (_backendAction.py:738-765, :810-919) with the busbars last registered.  A disconnected end is one <= 0.
        -> (aff_lines bool [B, n_line], aff_subs bool [B, n_sub]) of the LEGAL actions, applied to self.topo"""
        self._to_host()
        gm = self.gm
        lor, lex = self.line_or_pos, self.line_ex_pos
        live = ~self.done
        so, se = sb[:, lor], sb[:, lex]
        ch = cb[:, lor] | cb[:, lex]
        amb = ((sb != 0) & cb).any(axis=1) | ((ss != 0) & cs).any(axis=1)
        amb |= (((so == -1) & (se > 0)) | ((se == -1) & (so > 0))).any(axis=1)
        amb |= ((ss == -1) & ((so > 0) | (se > 0) | ch)).any(axis=1)
        amb |= ((ss == 1) & ((so == -1) | (se == -1) | ch)).any(axis=1)
        amb &= live
        # the impact: lines whose status is set, changed or reached through one end's busbar; substations of the other bus changes
        on = (self.topo[:, lor] > 0) & (self.topo[:, lex] > 0)
        named = cs | (ss != 0)
        conn = ((so > 0) | (se > 0)) & ~on
        disc = ((so < 0) | (se < 0)) & on
        aff_l = named | conn | disc
        clear = (named & ~on) | conn | disc
        eff = cb | (sb != 0)
        eff[:, lor] &= ~clear
        eff[:, lex] &= ~clear
        aff_s = (eff.astype(np.int64) @ self._pos_sub) > 0
        illegal = ~amb & self._illegal(aff_l, aff_s)
        self.is_illegal = illegal & live
        self.n_illegal += int(self.is_illegal.sum())
        self.is_ambiguous = amb
        ok = live & ~amb & ~illegal
        aff_l &= ok[:, None]
        aff_s &= ok[:, None]
        w = np.flatnonzero(ok & ((sb != 0).any(axis=1) | cb.any(axis=1) | (ss != 0).any(axis=1) | cs.any(axis=1)))
        if not len(w):
            return aff_l, aff_s

        def topo_stage(v, c, s):                                             # change_bus (connected: 1 <-> 2), then set_bus
            v = np.where(c & (v > 0), 3 - v, v)
            return np.where(s != 0, s, v)

        nt = gm.dim_topo
        t = self.topo[w, :nt].astype(np.int64)
        lb = self.last_bus[w].astype(np.int64)
        sbw, cbw, ssw, csw = sb[w].astype(np.int64), cb[w], ss[w], cs[w]
        lbo, lbe = lb[:, lor], lb[:, lex]
        vo, ve = t[:, lor], t[:, lex]
        was = (vo > 0) | (ve > 0)                                            # change_status, then set_status
        vo, ve = np.where(csw, np.where(was, -1, lbo), vo), np.where(csw, np.where(was, -1, lbe), ve)
        vo = np.where(ssw < 0, -1, np.where((ssw > 0) & (vo <= 0), lbo, vo))
        ve = np.where(ssw < 0, -1, np.where((ssw > 0) & (ve <= 0), lbe, ve))
        before_off = vo <= 0                                                 # _status_or_before
        disco = before_off | (ve <= 0)
        vo, ve = topo_stage(vo, cbw[:, lor], sbw[:, lor]), topo_stage(ve, cbw[:, lex], sbw[:, lex])
        reco = before_off & ((vo > 0) | (ve > 0))                            # _aux_iadd_reconcile_disco_reco
        off = ~reco & (disco | (vo <= 0) | (ve <= 0))
        vo = np.where(reco & (vo <= 0), lbo, np.where(off, -1, vo))
        ve = np.where(reco & (ve <= 0), lbe, np.where(off, -1, ve))
        t = topo_stage(t, cbw, sbw)
        t[:, lor], t[:, lex] = vo, ve
        self.topo[w, :nt] = t
        self.last_bus[w] = np.where(t > 0, t, lb)                            # last_topo_registered.update_connected
        self._topo_dirty = True
        self._cap_dirty[w] = True
        return aff_l, aff_s

    def _vector_action(self, set_bus, change_bus, set_line_status, change_line_status):
        """the four vectors of :meth:`step` checked and completed with zeros -> (set_bus int8 [B, dim_topo], change_bus bool
        [B, dim_topo], set_line_status int8 [B, n_line], change_line_status bool [B, n_line]), or None when none is given"""
        if set_bus is None and change_bus is None and set_line_status is None and change_line_status is None:
            return None
        gm, B = self.gm, self.batch
        out = []
        for x, name, n, kinds in ((set_bus, "set_bus", gm.dim_topo, "iu"), (change_bus, "change_bus", gm.dim_topo, "b"),
                                  (set_line_status, "set_line_status", gm.n_line, "iu"),
                                  (change_line_status, "change_line_status", gm.n_line, "b")):
            if x is None:
                out.append(np.zeros((B, n), dtype=bool if kinds == "b" else np.int8))
                continue
            x = np.asarray(x)
            if x.shape != (B, n) or x.dtype.kind not in kinds:
                raise ValueError(f"{name} must be a {'bool' if kinds == 'b' else 'int8'} array of shape {(B, n)}")
            out.append(x.astype(bool) if kinds == "b" else x)
        sb, cb, ss, cs = out
        if ((sb < -1) | (sb > gm.n_busbar)).any():
            raise ValueError(f"set_bus outside [-1, {gm.n_busbar}]")
        if ((sb == -1) & (self.line_of_pos < 0)[None, :]).any():
            raise ValueError("set_bus = -1 on a load, generator or storage unit (detachment is not supported)")
        if cb.any() and gm.n_busbar != 2:
            raise ValueError("change_bus needs two busbars per substation")
        if ((ss < -1) | (ss > 1)).any():
            raise ValueError("set_line_status outside {-1, 0, 1}")
        return sb.astype(np.int8), cb, ss.astype(np.int8), cs

    def set_action_table(self, table):
        """Bind a discrete action table (:class:`grid2op_b200.action_table.ActionTable`, checked when it was built): ``step`` /
        ``step_tensors(action_id=...)`` then act with row ``action_id[i]`` in instance i.  On the tensor path the library copies the
        table to the device once.  A new call replaces the table; one built for another grid raises ValueError."""
        if not table.matches(self.gm):
            raise ValueError(f"action table for another grid (dim_topo {table.dim_topo}, n_line {table.n_line}, {table.n_busbar} busbars)")
        if self._dev is not None:
            self.engine.act_table_bind(table.set_bus, table.change_bus, table.set_line_status, table.change_line_status)
        self._table = table

    def _table_rows(self, action_id):
        """``action_id`` int [B] checked against the bound table -> its rows (set_bus, change_bus, set_line_status,
        change_line_status)"""
        if self._table is None:
            raise ValueError("action_id without an action table (set_action_table)")
        a = np.asarray(action_id)
        if a.shape != (self.batch,) or a.dtype.kind not in "iu":
            raise ValueError(f"action_id must be an int array of shape {(self.batch,)}")
        if ((a < 0) | (a >= self._table.n)).any():
            raise ValueError(f"action_id outside [0, {self._table.n})")
        t = self._table
        return t.set_bus[a], t.change_bus[a], t.set_line_status[a], t.change_line_status[a]

    def _isolated_shunt_busbar(self) -> np.ndarray:
        """bool [B]: busbar 1 of a substation whose shunt is out of service in the grid file carries no element any more — for the
        reference an in-service bus without a voltage: ``runpf`` fails with "Isolated bus" (pandaPowerBackend.py:1241-1244) and the
        episode ends (baseEnv.py:3523-3524)."""
        if self._iso_cols is None:            # one gather over the positions of those substations + a segmented "any"
            keep = [pos for pos, other in zip(self._shunt_off_pos, self._shunt_off_other) if not other]
            # (other: an in-service shunt / the hidden slack unit sits on that substation, never moved by this driver)
            self._iso_cols = np.concatenate(keep) if keep else np.zeros(0, dtype=np.int64)
            self._iso_seg = np.cumsum([0] + [len(p) for p in keep])[:-1]
        if len(self._iso_cols) == 0:
            return np.zeros(self.batch, dtype=bool)
        on1 = (self.topo[:, self._iso_cols] == 1).astype(np.uint8)
        return (np.add.reduceat(on1, self._iso_seg, axis=1) == 0).any(axis=1)

    def _apply_environment(self):
        """maintenance / hazards of the row every instance is about to solve: those lines are out"""
        gm = self.gm
        forced = None
        r = self.row % self.chron.shape[1]
        if self._maint is not None:
            forced = self._maint[self.scen, r]
        if self._haz is not None:
            h = self._haz[self.scen, r]
            forced = h if forced is None else (forced | h)
        if forced is None:
            return
        forced = forced & ~self.done[:, None]
        ii, ll = np.nonzero(forced)
        if len(ii):
            was_on = (self.topo[ii, self.line_or_pos[ll]] > 0) | (self.topo[ii, self.line_ex_pos[ll]] > 0)
            self.topo[ii, self.line_or_pos[ll]] = -1
            self.topo[ii, self.line_ex_pos[ll]] = -1
            if was_on.any():
                self._topo_dirty = True
                self._cap_dirty[ii[was_on]] = True

    def step(self, sub_id=None, sub_bus=None, line_id=None, line_status=None, from_reset: bool = False, raise_alert=None,
             raise_alarm=None, set_bus=None, change_bus=None, set_line_status=None, change_line_status=None, action_id=None):
        """One env.step of every instance.  ``sub_id`` int [B] (-1: none) with ``sub_bus`` int8 [B, >= max_sub_size] (busbar per
        element of that substation in topology-vector order, 0 = leave); ``line_id`` int [B] (-1: none) with ``line_status``
        int [B] (+1 reconnect / -1 disconnect); ``raise_alert`` bool [B, dim_alerts] (:meth:`enable_alerts`; None: no alert,
        ignored on a reset step); ``raise_alarm`` bool [B, dim_alarms] (:meth:`enable_alarms`; None: no alarm, ignored on a reset
        step).  Returns ``(rho [B, n_line], done [B], info)``; the full records stay on the device (:meth:`fetch`).

        grid2op's native topology action instead of the ``sub_id`` / ``line_id`` pair (any subset of the four, not together with
        that pair): ``set_bus`` int8 [B, dim_topo] in ``topo_vect`` order (0 leave, -1 disconnect a line end, 1..n_busbar),
        ``change_bus`` bool [B, dim_topo] (two busbars per substation only), ``set_line_status`` int8 [B, n_line] in {-1, 0, 1},
        ``change_line_status`` bool [B, n_line]; :meth:`_apply_actions` restates what grid2op does with them.  ``info["is_ambiguous"]``
        (bool [B]) then says which actions were replaced by "do nothing" as ambiguous.  A value out of range, ``set_bus = -1`` on a
        load, generator or storage unit, a wrong shape or dtype raise ValueError and change nothing.

        ``action_id`` int [B] instead of any of the above: instance i acts with row ``action_id[i]`` of the table
        :meth:`set_action_table` bound, as the vector action above (``info["is_ambiguous"]`` included).  An id outside [0, n),
        no bound table, a wrong shape or dtype raise ValueError and change nothing."""
        vec = self._vector_action(set_bus, change_bus, set_line_status, change_line_status)
        if vec is not None and (sub_id is not None or line_id is not None):
            raise ValueError("the vector action (set_bus, change_bus, set_line_status, change_line_status) replaces sub_id / line_id")
        if action_id is not None:
            if vec is not None or sub_id is not None or line_id is not None:
                raise ValueError("action_id replaces sub_id / line_id and the vector action")
            vec = self._table_rows(action_id)
        if raise_alert is not None:
            if self._alerts is None:
                raise ValueError("raise_alert without enable_alerts()")
            raise_alert = np.asarray(raise_alert)
            if raise_alert.shape != (self.batch, self._alerts.n) or raise_alert.dtype.kind not in "bui":
                raise ValueError(f"raise_alert must be a bool array of shape {(self.batch, self._alerts.n)}")
            raise_alert = raise_alert != 0
        if raise_alarm is not None:
            if self._alarms is None:
                raise ValueError("raise_alarm without enable_alarms()")
            raise_alarm = np.asarray(raise_alarm)
            if raise_alarm.shape != (self.batch, self._alarms.n) or raise_alarm.dtype.kind not in "bui":
                raise ValueError(f"raise_alarm must be a bool array of shape {(self.batch, self._alarms.n)}")
            raise_alarm = raise_alarm != 0
        self._to_host()
        gm = self.gm
        opp = None
        if self._opp is not None:             # the opponent decides on the line status and rho the previous step left
            opp = self._opponent_decide(from_reset)
        self.is_ambiguous = np.zeros(self.batch, dtype=bool)
        if from_reset:
            aff_l, aff_s = np.zeros((self.batch, gm.n_line), dtype=bool), np.zeros((self.batch, gm.n_sub), dtype=bool)
        elif vec is not None:
            aff_l, aff_s = self._apply_actions(*vec)
        else:
            aff_l, aff_s = self._apply_agent(sub_id, sub_bus, line_id, line_status)
        self._apply_environment()
        if opp is not None:                   # its attack lands after the agent's action and the environment's outages
            self._apply_attack(*opp)
        if self._topo_dirty:
            self.engine.series_set_topo(self.topo)
            self._topo_dirty = False
            if self.tight_cap:
                self.nb_cap = self._bus_cap()
        if from_reset:
            self.engine.series_next_is_reset()
        self.step_device()
        out, status, iters, rho = self.engine.series_fetch(want_out=False)
        disc = None
        if self.protections:
            st = self.engine.series_fetch_state()
            disc = st["disc_lines"]
            tripped = (disc >= 0) & ~self.done[:, None]
            ii, ll = np.nonzero(tripped)
            if len(ii):                       # _backend_action.update_state(disc_lines): the tripped lines stay out
                self.topo[ii, self.line_or_pos[ll]] = -1
                self.topo[ii, self.line_ex_pos[ll]] = -1
                # (the engine's own mirror of the series topology already holds them: no re-upload needed)
        if len(self._shunt_off):              # (after the trips of this step: the cascade's re-solves see them too, backend.py:1466-1521)
            iso = self._isolated_shunt_busbar()
            if iso.any():
                status = np.where(iso, 2, status).astype(status.dtype)          # ST_UNSUPPLIED: the reference's "Isolated bus"
        r = self.row % self.chron.shape[1]
        # ---- cooldowns (baseEnv.py:3352-3393, :2566-2597), in the reference's order --------------------------------------
        live = ~self.done
        lc = self.line_cooldown
        lc[(lc > 0) & live[:, None]] -= 1
        if disc is not None:
            lc[(disc >= 0) & live[:, None]] = self.cd_reco
        if self._maint is not None:
            mt, md = self._maint_time[self.scen, r], self._maint_dur[self.scen, r]
            first = (mt == 0) & live[:, None]
            lc[first] = np.maximum(lc[first], md[first])
        if self._haz_dur is not None:
            hd = self._haz_dur[self.scen, r]
            lc[live] = np.maximum(lc[live], hd[live])
        if not from_reset:
            if self.cd_line > 0:
                cond = aff_l & (lc < self.cd_line)
                lc[cond] = self.cd_line
            if self.cd_sub > 0:
                sc = self.sub_cooldown
                sc[(sc > 0) & live[:, None]] -= 1
                sc[aff_s] = self.cd_sub
        newly_done = live & (status != 0)
        alert_reward = None
        if self._alerts is not None:          # after the attack; an instance finished before the step keeps its alert state
            alert_reward = self._alerts.step(None if from_reset else raise_alert, opp[0] if opp is not None else None,
                                             live & (not from_reset), newly_done).copy()
        self.done |= newly_done
        self.row = self.row + 1
        self.n_steps += 1
        if from_reset:
            self.is_illegal = np.zeros(self.batch, dtype=bool)
            self.current_step[live] = 0
            if self._obs is not None:
                self._obs["reset"][live] = True
        else:
            self.current_step[live] += 1
        alarm_reward = None
        if self._alarms is not None:          # registered once the step's legality is known; an instance finished before keeps its state
            alarm_reward = self._alarms.step(None if from_reset else raise_alarm, live & (not from_reset), self.is_illegal | self.is_ambiguous,
                                             self.current_step, newly_done, disc).copy()
        info = {"status": status, "iters": iters, "disc_lines": disc, "newly_done": newly_done, "is_illegal": self.is_illegal.copy()}
        if vec is not None:
            info["is_ambiguous"] = self.is_ambiguous.copy()
        if opp is not None:
            info["opponent_attack_line"], info["opponent_attack_duration"] = opp
        if alert_reward is not None and self._alerts.reward:
            info["rewards"] = {"alert": alert_reward}
        if alarm_reward is not None:
            info["is_alarm_illegal"] = self._alarms.s["illegal"].astype(bool)
            if self._alarms.reward:
                info["rewards"] = {"alarm": alarm_reward}
        return rho, self.done.copy(), info

    # ---- line alerts ------------------------------------------------------------------------------------------------------
    def enable_alerts(self, alertable_lines, *, alert_time_window: int = 12, reward: bool = True, reward_min_no_blackout: float = -1.0,
                      reward_min_blackout: float = -10.0, reward_max_no_blackout: float = 1.0, reward_max_blackout: float = 2.0,
                      reward_end_episode_bonus: float = 1.0):
        """grid2op's line alerts (l2rpn_idf_2023) for every instance: ``alertable_lines``, names (``GridModel.name_line``) or ids
        in grid2op's order (a list of areas, as the config's ``lines_attacked``, is flattened), at most 64; ``alert_time_window``:
        the ``ALERT_TIME_WINDOW`` parameter; ``reward``: compute ``AlertReward`` with these constants into
        ``info["rewards"]["alert"]`` (float64 [B], 0 for an instance finished before the step) and ``was_alert_used_after_attack``.
        The attacked lines are those of the opponent :meth:`enable_opponent` binds (none without one).  From then on :meth:`step`
        / :meth:`step_tensors` take ``raise_alert``, and :meth:`observe` fills the seven alert attributes.  Call it before
        :meth:`enable_observation` (the vector's width depends on ``dim_alerts``).  ``reward_end_episode_bonus`` is kept but never
        paid: this environment has no end of chronics, the caller resets."""
        from .alert import BatchedAlerts
        if self._obs is not None:
            raise RuntimeError("enable_alerts() before enable_observation(): the observation width depends on dim_alerts")
        if self._alarms is not None:
            raise ValueError("alerts and alarms are exclusive (an environment's alerts_info.json has \"by_line\" or \"fixed\")")
        names = list(getattr(self.gm, "name_line", []))
        flat = []
        for x in alertable_lines:
            flat.extend(x if isinstance(x, (list, tuple)) else [x])
        if len(flat) > 64:
            raise ValueError("more than 64 alertable lines")
        ids = []
        for x in flat:
            if isinstance(x, str):
                if x not in names:
                    raise ValueError(f"unknown line {x!r}")
                ids.append(names.index(x))
            else:
                ids.append(int(x))
        if not ids or any(not 0 <= l < self.gm.n_line for l in ids):
            raise ValueError("alertable line out of range (or no line)")
        if len(set(ids)) != len(ids):
            raise ValueError("alertable line listed twice")
        if int(alert_time_window) <= 0:
            raise ValueError("alert_time_window must be >= 1")
        self._to_host()
        self._alerts = BatchedAlerts(ids, self.batch, window=int(alert_time_window), reward=reward,
                                     reward_min_no_blackout=reward_min_no_blackout, reward_min_blackout=reward_min_blackout,
                                     reward_max_no_blackout=reward_max_no_blackout, reward_max_blackout=reward_max_blackout,
                                     reward_end_episode_bonus=reward_end_episode_bonus)
        if self._dev is not None:
            self._alert_bind_device()
        return self._alerts.n

    def alert_state(self) -> dict:
        """the alert state of every instance as the device keeps it (:data:`grid2op_b200.alert.ALERT_STATE`): last_alert, already
        (_is_already_attacked) uint8 [B, n]; tsl_alert, duration, tsl_attack, under_alert, was_used int32 [B, n]; total int32
        [B]; AlertReward's ts_attack / launched uint8 [B, window + 2, n], current uint8 [B, n] and cur_id int32 [B]"""
        if self._alerts is None:
            raise RuntimeError("call enable_alerts() first")
        self._to_host()
        return self._alerts.get_state()

    # ---- alarms -----------------------------------------------------------------------------------------------------------
    def enable_alarms(self, zones, *, max_budget: float = 3.0, budget_per_ts: float = 1.0 / 192, alarm_cost: float = 1.0,
                      init_budget: float = 2.0, alarm_best_time: int = 12, alarm_window_size: int = 12, reward: bool = True):
        """grid2op's alarms (l2rpn_icaps_2021) for every instance: ``zones`` the ``(names, zone mask per line)`` pair
        :func:`grid2op_b200.alarm.load_alarm_zones` reads from the environment's ``alerts_info.json``; the
        ``LinearAttentionBudget`` constants of the environment's ``kwargs_attention_budget``; ``alarm_best_time`` /
        ``alarm_window_size``: the ``ALARM_BEST_TIME`` / ``ALARM_WINDOW_SIZE`` parameters; ``reward``: compute ``AlarmReward`` into
        ``info["rewards"]["alarm"]`` (float64 [B], 0 for an instance finished before the step, non-zero only on the step that ends
        an episode).  From then on :meth:`step` / :meth:`step_tensors` take ``raise_alarm``, ``info["is_alarm_illegal"]`` (bool [B])
        says which alarms the budget refused, and :meth:`observe` fills the five alarm attributes.  Call it before
        :meth:`enable_observation` (the vector's width depends on ``dim_alarms``).  Alarms and alerts are exclusive; a ring of
        ``alarm_best_time + alarm_window_size`` steps is kept per instance, at most 1024.  AlarmReward's ``reward_max`` at the end
        of the chronics is never paid: this environment has no end of chronics, the caller resets."""
        from .alarm import MAX_RING, MAX_ZONES, BatchedAlarms
        if self._obs is not None:
            raise RuntimeError("enable_alarms() before enable_observation(): the observation width depends on dim_alarms")
        if self._alerts is not None:
            raise ValueError("alerts and alarms are exclusive (an environment's alerts_info.json has \"by_line\" or \"fixed\")")
        names, mask = zones
        mask = np.asarray(mask)
        n = len(names)
        if not 1 <= n <= MAX_ZONES:
            raise ValueError(f"{n} alarm zones, 1 to {MAX_ZONES} supported")
        if mask.shape != (self.gm.n_line,) or mask.dtype.kind not in "ui" or (mask <= 0).any() or (mask >= 2 ** n).any():
            raise ValueError(f"the zone masks must be {self.gm.n_line} integers, each line in at least one of the {n} zones")
        best, win = int(alarm_best_time), int(alarm_window_size)
        if best <= 0 or win <= 0:
            raise ValueError("alarm_best_time and alarm_window_size must be >= 1")
        if best + win > MAX_RING:
            raise ValueError(f"alarm_best_time + alarm_window_size must be <= {MAX_RING}")
        self._to_host()
        self._alarms = BatchedAlarms(mask, n, self.batch, max_budget=max_budget, budget_per_ts=budget_per_ts, alarm_cost=alarm_cost,
                                     init_budget=init_budget, best_time=best, window_size=win, reward=reward)
        self._alarms.names = list(names)
        if self._dev is not None:
            self._alarm_bind_device()
        return n

    def alarm_state(self) -> dict:
        """the alarm state of every instance as the device keeps it (:data:`grid2op_b200.alarm.ALARM_STATE`): budget float32 [B];
        time_last, time_last_ok int32 [B]; last, last_ok int32 [B, n_zone]; the ring of successful alarms ring_step int32 /
        ring_mask uint32 [B, best_time + window_size]; any_ok, used (AlarmReward.is_alarm_used), illegal uint8 [B]"""
        if self._alarms is None:
            raise RuntimeError("call enable_alarms() first")
        self._to_host()
        return self._alarms.get_state()

    # ---- line-attack opponent ---------------------------------------------------------------------------------------------
    def enable_opponent(self, kind: str, lines_attacked, *, attack_duration: int, attack_cooldown: int, budget_per_ts: float,
                        init_budget: float, attack_period: Optional[int] = None, rho_normalization=None, seeds,
                        attack_every_xxx_hour: Optional[float] = None, average_attack_duration_hour: Optional[float] = None,
                        minimum_attack_duration_hour: Optional[float] = None, pmax_pmin_ratio: float = 4,
                        delta_time_seconds: float = 300.0, episode_max_time=None):
        """Give every instance grid2op's line-attack opponent (``OpponentSpace`` + ``BaseActionBudget``): ``kind``
        ``"RandomLineOpponent"``, ``"WeightedRandomOpponent"`` or ``"GeometricOpponent"``; ``lines_attacked``: line names
        (``GridModel.name_line``) or ids; the other parameters are the environment config's ``opponent_attack_duration``,
        ``opponent_attack_cooldown``, ``opponent_budget_per_ts``, ``opponent_init_budget`` and ``kwargs_opponent``
        (``attack_period``, ``rho_normalization``; ``attack_every_xxx_hour``, ``average_attack_duration_hour``,
        ``minimum_attack_duration_hour``, ``pmax_pmin_ratio`` for the GeometricOpponent, with the environment's
        ``delta_time_seconds``); ``seeds``: int [B], the opponent seed of each instance (:func:`grid2op_b200.opponent.opponent_seed`
        of an environment seed gives the one ``env.seed`` gives).  Every instance starts from ``OpponentSpace.reset()``, the
        GeometricOpponent with the attack schedule ``env.seed(s); env.reset()`` draws; :meth:`reset_instances` resets it again (its
        random stream continues, a new schedule is drawn).  ``episode_max_time`` (GeometricOpponent): ``env.max_episode_duration()``,
        an int or one per scenario of the chronics array; default: the scenarios' ``max_step`` when :meth:`enable_observation` was
        called first, else the chronics array's row count - 1.  Call it after the first step (``reset_step``): the weighted and
        geometric opponents read the rho of the previous step.  From then on :meth:`step` / :meth:`step_tensors` report
        ``info["opponent_attack_line"]`` (int32 [B], -1: none) and ``info["opponent_attack_duration"]`` (int32 [B]).

        ``"GeometricOpponentMultiArea"`` (l2rpn_idf_2023): ``lines_attacked`` is a list of areas (lists of names or ids), at most 8
        areas and 64 lines, no line in two areas; the other arguments are the GeometricOpponent's, and ``attack_cooldown`` must be 0
        or 1.  Each area is a GeometricOpponent with its own stream (seeded from the instance's seed as ``env.seed`` seeds it) and
        schedule; ``info["opponent_attack_line"]`` is then int32 [B, n_area], each area's line in the step's attack (-1: none), and
        ``info["opponent_attack_duration"]`` is 1 where an attack landed."""
        from .opponent import BatchedOpponent
        if self.n_steps == 0:
            raise RuntimeError("enable_opponent() after the first step (reset_step): the opponent observes the previous step")
        self._to_host()
        names = list(getattr(self.gm, "name_line", []))

        def line_ids(group):
            ids = [names.index(x) if isinstance(x, str) else int(x) for x in group]
            if any(not 0 <= l < self.gm.n_line for l in ids):
                raise ValueError("attacked line out of range")
            return ids
        ids = [line_ids(a) for a in lines_attacked] if kind == "GeometricOpponentMultiArea" else line_ids(lines_attacked)
        geo = {}
        if kind in ("GeometricOpponent", "GeometricOpponentMultiArea"):
            if episode_max_time is None:
                per_scen = (self._obs["tables"]["max_step"] if self._obs is not None
                            else np.full(self.chron.shape[0], self.chron.shape[1] - 1))
            else:
                per_scen = np.broadcast_to(np.asarray(episode_max_time, dtype=np.int64), (self.chron.shape[0],))
            geo = dict(attack_every_xxx_hour=attack_every_xxx_hour, average_attack_duration_hour=average_attack_duration_hour,
                       minimum_attack_duration_hour=minimum_attack_duration_hour, pmax_pmin_ratio=pmax_pmin_ratio,
                       delta_time_seconds=delta_time_seconds, episode_max_time=np.asarray(per_scen, dtype=np.int64)[self.scen])
        self._opp = BatchedOpponent(kind, ids, self.batch, attack_duration=attack_duration, attack_cooldown=attack_cooldown,
                                    budget_per_ts=budget_per_ts, init_budget=init_budget, seeds=seeds, attack_period=attack_period,
                                    rho_normalization=rho_normalization, **geo)
        if self._dev is not None:
            self._opp_bind_device()

    def _opponent_decide(self, from_reset):
        """OpponentSpace.attack of the live instances (none on a reset step) -> (line int32 [B], duration int32 [B])"""
        o = self._opp
        if from_reset:
            line = np.full((self.batch, len(o.area_off) - 1) if o.multi else self.batch, -1, dtype=np.int32)
            return line, np.zeros(self.batch, dtype=np.int32)
        rho = (self.engine.series_fetch(want_out=False)[3] if o.weighted or o.geometric or o.multi
               else None)                                                   # (what the previous step wrote)
        return o.attack(self.line_status(), rho, ~self.done)

    def _apply_attack(self, line, dur):
        """the attacked lines are out (both ends), their cooldown at least the attack's duration (``line`` [B] or, several lines
        per instance, [B, n])"""
        ii, kk = np.nonzero(line.reshape(self.batch, -1) >= 0)
        if not len(ii):
            return
        ll = line.reshape(self.batch, -1)[ii, kk].astype(np.int64)
        lc = self.line_cooldown
        lc[ii, ll] = np.maximum(lc[ii, ll], dur[ii])
        was_on = (self.topo[ii, self.line_or_pos[ll]] > 0) | (self.topo[ii, self.line_ex_pos[ll]] > 0)
        self.topo[ii, self.line_or_pos[ll]] = -1
        self.topo[ii, self.line_ex_pos[ll]] = -1
        if was_on.any():
            self._topo_dirty = True
            self._cap_dirty[ii[was_on]] = True

    def opponent_state(self) -> dict:
        """the opponent state of every instance as the device keeps it: budget float64 [B], budget64 uint8 [B] (the budget is a
        float64 since its first charge), ctr int32 [B, 4] (attack duration, cooldown, last line, steps to the weighted opponent's
        next attack), mt uint32 [B, 624] / mt_pos int32 [B] (the random streams); a GeometricOpponent adds geo_wait / geo_dur
        int32 [B, cap] (its attack schedules) and geo_ctr int32 [B, 4] (schedule length, attacks consumed, previous_fails, schedule
        entries dropped at the cap: 0 unless the cap was too small); a GeometricOpponentMultiArea adds multi_mt / multi_mt_pos,
        multi_wait / multi_dur, multi_ctr and multi_fails (:meth:`grid2op_b200.opponent.BatchedOpponent.get_state`)"""
        if self._opp is None:
            raise RuntimeError("call enable_opponent() first")
        self._to_host()
        return self._opp.get_state()

    def line_angles(self, out: np.ndarray):
        """``theta_or, theta_ex`` [B, n_line] of the full result records ``out`` (:meth:`fetch`) as an OBSERVATION of the reference
        shows them: the kernels' records carry 0 for open lines, PandaPowerBackend reports the angle of the bus the end was last
        attached to (it zeroes the voltage of open lines, not the angle: pandaPowerBackend.py:1163-1187), 0 when that busbar has no
        element left.  Same rule as ``B200Backend._theta_of_open_lines``, for the whole batch."""
        from .engine import OutputView
        self._to_host()
        gm, B = self.gm, self.batch
        v = OutputView(gm, out)
        th_or, th_ex = np.array(v.theta_or, dtype=np.float32), np.array(v.theta_ex, dtype=np.float32)
        on = self.line_status()
        if on.all():
            return th_or, th_ex
        ns, nh, dt = gm.n_sub, gm.n_hidden, gm.dim_topo
        slot_theta = np.full((B, gm.n_slot + 1), np.nan, dtype=np.float64)          # (last column: dump for disconnected elements)

        def scatter(sub, pos, theta):
            bus = self.topo[:, pos].astype(np.int64)
            slot = np.where(bus > 0, np.asarray(sub, dtype=np.int64)[None, :] + (bus - 1) * ns, gm.n_slot)
            np.put_along_axis(slot_theta, slot, np.asarray(theta, dtype=np.float64), axis=1)

        scatter(gm.line_or_sub, self.line_or_pos, v.theta_or); scatter(gm.line_ex_sub, self.line_ex_pos, v.theta_ex)
        scatter(gm.gen_sub, np.asarray(gm.gen_pos, dtype=np.int64), v.unit_theta[:, nh:])
        scatter(gm.load_sub, np.asarray(gm.load_pos, dtype=np.int64), v.load_theta)
        slot_theta[:, gm.n_slot] = np.nan
        for th, sub, pos in ((th_or, gm.line_or_sub, self.line_or_pos), (th_ex, gm.line_ex_sub, self.line_ex_pos)):
            last = self.last_bus[:, pos].astype(np.int64)
            a = np.take_along_axis(slot_theta, np.asarray(sub, dtype=np.int64)[None, :] + (last - 1) * ns, axis=1)
            th[~on] = np.where(np.isfinite(a), a, 0.0)[~on]
        return th_or, th_ex

    def reset_instances(self, idx, rows=None):
        """``env.reset()`` of the instances ``idx`` (typically the finished ones): plain topology, cooldowns / counters / done flag
        cleared on the host and on the device, next chronics row ``rows`` (default: the row each instance started from).  Their
        next :meth:`step` is an ordinary step on that row (use ``rows - 1`` semantics of your agent loop accordingly).
        ``idx`` may also be a CUDA bool mask [B] (``rows``: None or a CUDA integer tensor [B]): the reset then runs on the device
        (:meth:`step_tensors`)."""
        if _is_cuda_tensor(idx):
            return self._reset_tensors(idx, rows)
        self._to_host()
        idx = np.asarray(idx, dtype=np.int64)
        if len(idx) == 0:
            return
        rows = self.t0[idx].astype(np.int64) if rows is None else np.asarray(rows, dtype=np.int64)
        self.topo[idx] = self.topo0[idx]
        self.last_bus[idx] = np.where(self.topo0[idx, :self.gm.dim_topo] > 0, self.topo0[idx, :self.gm.dim_topo], 1)
        self.line_cooldown[idx] = 0; self.sub_cooldown[idx] = 0
        self.done[idx] = False
        self.current_step[idx] = 0; self.is_illegal[idx] = False; self.is_ambiguous[idx] = False
        if self._obs is not None:
            self._obs["reset"][idx] = True
        self.row[idx] = rows
        if self._opp is not None:
            self._opp.reset(idx)
        if self._alerts is not None:
            self._alerts.reset(idx)
        if self._alarms is not None:
            self._alarms.reset(idx)
        self.engine.series_reset_instances(idx, t_new=rows % self.chron.shape[1], topo_rows=self.topo[idx])
        self._cap_dirty[idx] = True
        if self.tight_cap:
            self.nb_cap = self._bus_cap()

    # ---- observation layer ---------------------------------------------------------------------------------------------
    def enable_observation(self, env_dir: str, attrs=None, reward: Optional[str] = "RedispReward", scenarios=None,
                           init_storage_capacity: float = 0.5, activate_storage_loss: bool = True):
        """Let :meth:`observe` assemble grid2op observation vectors (``obs.to_vect()`` of the attribute list ``attrs``, default
        ``CompleteObservation.attr_list_vect``; pass the environment's own observation class list or a gym-style subset) and
        rewards (``"RedispReward"``, ``"L2RPNReward"`` or None) on the device.  ``env_dir``: the environment folder
        (``prods_charac.csv``, ``storage_units_charac.csv``, ``chronics/``); ``scenarios``: the chronics folders in the order of
        the ``chron`` array (default: every folder of ``env_dir/chronics``, sorted, as :func:`chronics.load_scenarios` reads them)."""
        from . import observation as ob
        from .chronics import list_scenarios
        if reward not in ob.REWARDS:
            raise ValueError(f"unknown reward class {reward!r} (RedispReward, L2RPNReward or None)")
        gm = self.gm
        n_alert = self._alerts.n if self._alerts is not None else 0
        n_alarm = self._alarms.n if self._alarms is not None else 0
        seg, n_obs = ob.obs_spec(gm, attrs, n_alert, n_alarm)
        folders = list(scenarios) if scenarios is not None else list_scenarios(os.path.join(env_dir, "chronics"))
        if len(folders) != self.chron.shape[0]:
            raise ValueError(f"{len(folders)} scenario folders for {self.chron.shape[0]} scenarios of the chronics array")
        cal, dt_min, max_step = ob.load_calendar(folders, self.chron.shape[1])
        gen = ob.load_gen_charac(env_dir, gm)
        if reward == "RedispReward" and not gen["available"]:
            raise ValueError("RedispReward needs the generator costs of prods_charac.csv")
        t = dict(seg=seg, n_obs=n_obs, calendar=cal, max_step=max_step, delta_time=dt_min, gen=gen,
                 storage=ob.load_storage(env_dir, gm, dt_min, init_storage_capacity, activate_storage_loss),
                 maint_time=self._maint_time, maint_dur=self._maint_dur, reward_kind=ob.REWARDS[reward],
                 reward=ob.reward_constants(gen, dt_min) if gen["available"] else dict(max_regret=0.0, reward_min=0.0, reward_illegal=0.0,
                                                                                       dts_hours=dt_min / 60.0),
                 soft_thr=self.soft_overflow_threshold, n_alert=n_alert, n_alarm=n_alarm)
        if reward == "L2RPNReward":
            t["reward"]["reward_min"] = 0.0
        self.engine.obs_bind(t)
        self._obs = dict(tables=t, n_obs=n_obs, reward=reward, reset=np.ones(self.batch, dtype=bool),
                         host_in=np.zeros((self.batch, gm.n_line + gm.n_sub + 3 + (6 * n_alert + 1 if n_alert else 0) +
                                           (n_alarm + 4 if n_alarm else 0)), dtype=np.int32))
        return n_obs

    def observe_inputs(self) -> np.ndarray:
        """int32 [B, n_line + n_sub + 3]: the per-instance values only the host knows (cooldowns, current_step, step stamp, flags
        illegal / game over / reset / ambiguous) — what one observe launch copies to the device; with alerts, 6 dim_alerts + 1 more columns
        (the alert values, :meth:`grid2op_b200.alert.BatchedAlerts.obs_record`); with alarms, dim_alarms + 4 more (the alarm values,
        :meth:`grid2op_b200.alarm.BatchedAlarms.obs_record`)."""
        self._to_host()
        gm, o = self.gm, self._obs
        h = o["host_in"]
        nl, ns = gm.n_line, gm.n_sub
        h[:, :nl] = self.line_cooldown; h[:, nl:nl + ns] = self.sub_cooldown
        h[:, nl + ns] = self.current_step; h[:, nl + ns + 1] = self.n_steps
        h[:, nl + ns + 2] = self.is_illegal * 1 + self.done * 2 + o["reset"] * 4 + self.is_ambiguous * 8
        if self._alerts is not None:
            h[:, nl + ns + 3:nl + ns + 4 + 6 * self._alerts.n] = self._alerts.obs_record()
        if self._alarms is not None:
            h[:, h.shape[1] - self._alarms.n - 4:] = self._alarms.obs_record(self.current_step)
        return h

    def observe(self, obs_out=None, reward_out=None):
        """grid2op observation vectors and rewards of the last step for the whole batch -> ``(obs [B, n_obs], reward [B])`` as torch
        CUDA tensors (``obs_out`` / ``reward_out``: caller-owned float32 tensors to write into).  One launch on the engine's stream
        behind the step; the result records never leave the device.  Call it once after every step: the overflow counters of the
        vector advance with it.  With a host-side engine (tests) numpy arrays come back."""
        if self._obs is None:
            raise RuntimeError("call enable_observation() first")
        B, n_obs = self.batch, self._obs["n_obs"]
        if self._authority == "device":
            return self._observe_device(obs_out, reward_out)
        host_in = self.observe_inputs()
        if not hasattr(self.engine, "h"):                 # host-side engine (test infrastructure): numpy in / out
            obs, rew = self.engine.observe_host(host_in, obs_out, reward_out)
            self._obs["reset"][:] = False
            return obs, rew
        import torch
        dev = torch.device("cuda", getattr(self.engine, "device", 0))
        obs = obs_out if obs_out is not None else torch.empty((B, n_obs), dtype=torch.float32, device=dev)
        rew = reward_out if reward_out is not None else torch.empty(B, dtype=torch.float32, device=dev)
        if obs.dtype != torch.float32 or tuple(obs.shape) != (B, n_obs) or not obs.is_cuda or not obs.is_contiguous():
            raise ValueError(f"obs_out must be a contiguous float32 CUDA tensor of shape {(B, n_obs)}")
        if rew.dtype != torch.float32 or tuple(rew.shape) != (B,) or not rew.is_cuda or not rew.is_contiguous():
            raise ValueError(f"reward_out must be a contiguous float32 CUDA tensor of shape {(B,)}")
        cur = torch.cuda.current_stream(obs.device)
        eng_stream = torch.cuda.ExternalStream(self.engine.stream, device=obs.device)
        eng_stream.wait_stream(cur)                       # (the tensors may have been written on torch's stream)
        self.engine.observe(host_in, obs.data_ptr(), rew.data_ptr())
        cur.wait_stream(eng_stream)                       # torch's consumers run behind the observe launch (no host sync)
        self._obs["reset"][:] = False
        return obs, rew

    def _observe_device(self, obs_out, reward_out):
        """:meth:`observe` in tensor mode: the input record the last step wrote on the device, no host copy"""
        import torch
        B, n_obs = self.batch, self._obs["n_obs"]
        dev = self._dev["device"]
        obs = obs_out if obs_out is not None else torch.empty((B, n_obs), dtype=torch.float32, device=dev)
        rew = reward_out if reward_out is not None else torch.empty(B, dtype=torch.float32, device=dev)
        _check_tensor(obs, "obs_out", (B, n_obs), (torch.float32,), dev)
        _check_tensor(rew, "reward_out", (B,), (torch.float32,), dev)
        if not (obs.is_contiguous() and rew.is_contiguous()):
            raise ValueError("obs_out / reward_out must be contiguous")
        cur, eng = self._streams()
        eng.wait_stream(cur)
        self.engine.observe_device(obs.data_ptr(), rew.data_ptr())
        cur.wait_stream(eng)
        return obs, rew

    # ---- tensor path: actions in, state out, as CUDA tensors ------------------------------------------------------------
    def _streams(self):
        import torch
        dev = self._dev["device"]
        return torch.cuda.current_stream(dev), torch.cuda.ExternalStream(self.engine.stream, device=dev)

    def _tensor_state(self):
        """the device buffers of the per-instance state, bound to the engine on first use"""
        if self._dev is not None:
            return self._dev
        if not hasattr(self.engine, "h"):
            raise RuntimeError("step_tensors needs the CUDA engine")
        import torch
        gm, B = self.gm, self.batch
        dev = torch.device("cuda", getattr(self.engine, "device", 0))
        z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)       # noqa: E731
        st = dict(last_bus=z((B, gm.dim_topo), torch.int8), line_cd=z((B, gm.n_line), torch.int32), sub_cd=z((B, gm.n_sub), torch.int32),
                  done=z(B, torch.bool), is_illegal=z(B, torch.bool), newly_done=z(B, torch.bool), current_step=z(B, torch.int32),
                  status=z(B, torch.int32), is_ambiguous=z(B, torch.bool))
        if self._iso_cols is None:
            self._isolated_shunt_busbar()                 # (builds the column segments)
        tables = dict(sub_pos=self.sub_pos, line_of_pos=self.line_of_pos, other_end_pos=self.other_end_pos, cd_line=self.cd_line,
                      cd_sub=self.cd_sub, cd_reco=self.cd_reco, maint=self._maint, haz=self._haz, maint_time=self._maint_time,
                      maint_dur=self._maint_dur, haz_dur=self._haz_dur, iso_seg=self._iso_seg, iso_cols=self._iso_cols,
                      topo0=self.topo0, t0=self.t0)
        self.engine.env_bind(tables, {k: v.data_ptr() for k, v in st.items() if k != "is_ambiguous"})
        # the rules, and the vector action's buffers: step_tensors copies the caller's tensors into them on the device
        st.update(act_set_bus=z((B, gm.dim_topo), torch.int8), act_change_bus=z((B, gm.dim_topo), torch.bool),
                  act_set_status=z((B, gm.n_line), torch.int8), act_change_status=z((B, gm.n_line), torch.bool))
        self.engine.act_bind(self.max_sub_changed, self.max_line_status_changed, 0 if self.areas is None else len(self.areas),
                             self._sub_area, self._line_area,
                             st["act_set_bus"].data_ptr(), st["act_change_bus"].data_ptr(), st["act_set_status"].data_ptr(),
                             st["act_change_status"].data_ptr(), st["is_ambiguous"].data_ptr())
        p, q = self.engine.series_device_pointers(), self.engine.env_pointers()
        st["rho"] = _device_view(p["rho"], (B, gm.n_line), "<f4", dev)
        st["iters"] = _device_view(p["iters"], (B,), "<i4", dev)
        st["disc"] = _device_view(q["disc"], (B, gm.n_line), "<i4", dev)
        st["device"] = dev
        self._dev = st
        self._illegal_seen = 0
        if self._table is not None:
            t = self._table
            self.engine.act_table_bind(t.set_bus, t.change_bus, t.set_line_status, t.change_line_status)
        if self._opp is not None:
            self._opp_bind_device()
        if self._alerts is not None:
            self._alert_bind_device()
        if self._alarms is not None:
            self._alarm_bind_device()
        return st

    def _opp_bind_device(self):
        """the opponent's constants and initial random states to the device; its per-step outputs are device buffers of ours"""
        import torch
        from .opponent import MULTI_KEYS
        d, o, B = self._dev, self._opp, self.batch
        z = lambda dt: torch.zeros(B, dtype=dt, device=d["device"])           # noqa: E731
        d["opp_line"], d["opp_dur"], d["opp_budget"] = z(torch.int32), z(torch.int32), z(torch.float64)
        s = o.get_state()
        self.engine.opp_bind(dict(kind=o.code, lines=o.lines, rho_norm=o.rho_norm, attack_period=o.attack_period,
                                  attack_duration=int(o.attack_duration), attack_cooldown=int(o.attack_cooldown),
                                  budget_per_ts=float(o.budget_per_ts), init_budget=float(o.init_budget), mt=s["mt"], mt_pos=s["mt_pos"]),
                             d["opp_line"].data_ptr(), d["opp_dur"].data_ptr(), d["opp_budget"].data_ptr())
        if o.geometric:
            self.engine.opp_geo_bind(dict(weights=o.geo_weights, p_hazard=o.hazard_rate, p_recovery=o.recovery_rate,
                                          logq_hazard=o.logq_hazard, logq_recovery=o.logq_recovery,
                                          recovery_min=o.recovery_min, episode_max_time=o.emt, geo_wait=s["geo_wait"],
                                          geo_dur=s["geo_dur"], geo_ctr=s["geo_ctr"]))
        if o.multi:
            d["opp_lines"] = torch.full((B, len(o.area_off) - 1), -1, dtype=torch.int32, device=d["device"])
            self.engine.opp_multi_bind(dict(area_off=o.area_off, weights=o.area_weights, p_hazard=o.hazard_rate,
                                            p_recovery=o.recovery_rate, logq_hazard=o.logq_hazard, logq_recovery=o.logq_recovery,
                                            recovery_min=o.recovery_min, episode_max_time=o.emt, **{k: s[k] for k in MULTI_KEYS}),
                                       d["opp_lines"].data_ptr())
        self._authority = "host"              # (the next step_tensors pushes the whole state, the opponent's included)

    def _alert_bind_device(self):
        """the alert constants to the device; the step's raise_alert and AlertReward are device buffers of ours"""
        import torch
        d, a, B = self._dev, self._alerts, self.batch
        d["alert_raise"] = torch.zeros((B, a.n), dtype=torch.uint8, device=d["device"])
        d["alert_reward"] = torch.zeros(B, dtype=torch.float64, device=d["device"])
        self.engine.alert_bind(a, d["alert_raise"].data_ptr(), d["alert_reward"].data_ptr())
        self._authority = "host"              # (the next step_tensors pushes the whole state, the alerts' included)

    def _alarm_bind_device(self):
        """the alarm constants to the device; the step's raise_alarm, AlarmReward and is_alarm_illegal are device buffers of ours"""
        import torch
        d, a, B = self._dev, self._alarms, self.batch
        d["alarm_raise"] = torch.zeros((B, a.n), dtype=torch.uint8, device=d["device"])
        d["alarm_reward"] = torch.zeros(B, dtype=torch.float64, device=d["device"])
        d["alarm_illegal"] = torch.zeros(B, dtype=torch.bool, device=d["device"])        # (written as uint8 0 / 1)
        self.engine.alarm_bind(a, d["alarm_raise"].data_ptr(), d["alarm_reward"].data_ptr(), d["alarm_illegal"].data_ptr())
        self._authority = "host"              # (the next step_tensors pushes the whole state, the alarms' included)

    def _to_device(self):
        """hand the host state to the tensor path"""
        import torch
        d = self._tensor_state()
        if self._authority == "device":
            return
        for name, arr in (("last_bus", self.last_bus), ("line_cd", self.line_cooldown), ("sub_cd", self.sub_cooldown), ("done", self.done),
                          ("is_illegal", self.is_illegal), ("current_step", self.current_step), ("is_ambiguous", self.is_ambiguous)):
            d[name].copy_(torch.from_numpy(np.ascontiguousarray(arr)))
        torch.cuda.current_stream(d["device"]).synchronize()
        obs = self._obs is not None
        self.engine.env_set_state(self.topo, self._nb_inst, self._cap_dirty, self._obs["reset"] if obs else None,
                                  self.observe_inputs() if obs else None)
        if self._opp is not None:
            s = self._opp.get_state()
            self.engine.opp_set_state(s)
            if self._opp.geometric:
                self.engine.opp_geo_set_state(s)
            if self._opp.multi:
                self.engine.opp_multi_set_state(s)
        if self._alerts is not None:
            self.engine.alert_set_state(self._alerts.get_state())
        if self._alarms is not None:
            self.engine.alarm_set_state(self._alarms.get_state())
        self._illegal_seen = self.engine.env_stats()["n_illegal"]
        self._authority = "device"

    def _to_host(self):
        """hand the tensor path's state to the host path"""
        if self._authority != "device":
            return
        d = self._dev
        s = self.engine.env_get_state()                   # (waits for the engine's stream)
        self._authority = "host"
        self.topo[:] = s["topo"]
        self.row = s["t"].astype(np.int64)
        self.last_bus[:] = d["last_bus"].cpu().numpy(); self.line_cooldown[:] = d["line_cd"].cpu().numpy()
        self.sub_cooldown[:] = d["sub_cd"].cpu().numpy(); self.done[:] = d["done"].cpu().numpy()
        self.is_illegal = d["is_illegal"].cpu().numpy().copy(); self.current_step[:] = d["current_step"].cpu().numpy()
        self.is_ambiguous = d["is_ambiguous"].cpu().numpy().copy()
        self._nb_inst[:] = s["nb_inst"]; self._cap_dirty[:] = s["cap_dirty"]
        if self._obs is not None:
            self._obs["reset"][:] = s["obs_reset"]
        if self._opp is not None:
            s = self.engine.opp_get_state()
            if self._opp.geometric:
                s.update(self.engine.opp_geo_get_state())
            if self._opp.multi:
                s.update(self.engine.opp_multi_get_state())
            self._opp.set_state(s)
        if self._alerts is not None:
            self._alerts.set_state(self.engine.alert_get_state())
            self._alerts.reward_out[:] = self._dev["alert_reward"].cpu().numpy()
        if self._alarms is not None:
            self._alarms.set_state(self.engine.alarm_get_state())
            self._alarms.reward_out[:] = self._dev["alarm_reward"].cpu().numpy()
        if self.tight_cap and self._cap_dirty.any():
            self.nb_cap = self._bus_cap()

    def step_tensors(self, sub_id=None, sub_bus=None, line_id=None, line_status=None, from_reset: bool = False, raise_alert=None,
                     raise_alarm=None, set_bus=None, change_bus=None, set_line_status=None, change_line_status=None, action_id=None):
        """:meth:`step` with the actions as CUDA tensors and the state kept on the device: ``sub_id`` int32 / int64 [B] (-1: none)
        with ``sub_bus`` int8 / int32 / int64 [B, >= max_sub_size]; ``line_id`` int32 / int64 [B] (-1: none) with ``line_status``
        int32 / int64 [B] (> 0 reconnect / < 0 disconnect).  Same semantics and bit-identical state as :meth:`step`; ordered against torch's current
        stream.  Returns ``(rho [B, n_line], done [B], info)`` as CUDA tensors; ``info``: ``status`` (with the isolated-busbar
        override), ``iters``, ``newly_done``, ``is_illegal``, ``disc_lines`` (protections on, else None).  The returned tensors
        are the environment's own buffers: the next step overwrites them.  The host waits once per step for a few words (and
        copies back the changed topology rows when the plans have to be looked up, which waits again).  An id or busbar out of
        range raises ValueError and changes nothing.  ``raise_alert``: bool / uint8 CUDA tensor [B, dim_alerts] (:meth:`enable_alerts`;
        None: no alert); ``info["rewards"]["alert"]`` is then the environment's float64 [B] buffer of the AlertReward.
        ``raise_alarm``: bool / uint8 CUDA tensor [B, dim_alarms] (:meth:`enable_alarms`; None: no alarm); ``info["rewards"]["alarm"]``
        and ``info["is_alarm_illegal"]`` are then the environment's float64 / bool [B] buffers.
        The vector action of :meth:`step` as CUDA tensors: ``set_bus`` int8 [B, dim_topo], ``change_bus`` bool [B, dim_topo],
        ``set_line_status`` int8 [B, n_line], ``change_line_status`` bool [B, n_line] (any subset, not with sub_id / line_id), copied
        on the device into the environment's buffers; ``info["is_ambiguous"]`` is then its bool [B] buffer.  A value out of range
        raises ValueError from the validation launch and changes nothing.
        ``action_id``: int32 / int64 CUDA tensor [B] instead of any of the above, ids into the table :meth:`set_action_table` bound
        (copied to the device once, at the bind); each instance reads its own row inside the step's launches.  An id outside
        [0, n) raises ValueError from the validation launch and changes nothing."""
        import torch
        d = self._tensor_state()
        dev, B = d["device"], self.batch
        if (sub_id is None) != (sub_bus is None) or (line_id is None) != (line_status is None):
            raise ValueError("sub_id / sub_bus and line_id / line_status come in pairs")
        gm = self.gm
        vec = [(set_bus, "set_bus", (B, gm.dim_topo), torch.int8), (change_bus, "change_bus", (B, gm.dim_topo), torch.bool),
               (set_line_status, "set_line_status", (B, gm.n_line), torch.int8),
               (change_line_status, "change_line_status", (B, gm.n_line), torch.bool)]
        use_vec = any(x is not None for x, _, _, _ in vec)
        if use_vec:
            if sub_id is not None or line_id is not None:
                raise ValueError("the vector action (set_bus, change_bus, set_line_status, change_line_status) replaces sub_id / line_id")
            for x, name, shape, dt in vec:
                if x is not None:
                    _check_tensor(x, name, shape, (dt,), dev)
            if change_bus is not None and gm.n_busbar != 2:
                raise ValueError("change_bus needs two busbars per substation")
        if action_id is not None:
            if use_vec or sub_id is not None or line_id is not None:
                raise ValueError("action_id replaces sub_id / line_id and the vector action")
            if self._table is None:
                raise ValueError("action_id without an action table (set_action_table)")
        ints = (torch.int32, torch.int64)
        keep = []

        def ids(x, name):
            _check_tensor(x, name, (B,), ints, dev)
            y = x if x.dtype == torch.int32 else x.clamp(-2 ** 31, 2 ** 31 - 1).to(torch.int32)   # (out of range stays out of range)
            y = y.contiguous()
            keep.append(y)
            return y.data_ptr()

        sid = sbus = lid = lst = 0
        cols = stride = 0
        if sub_id is not None:
            sid = ids(sub_id, "sub_id")
            if not (torch.is_tensor(sub_bus) and sub_bus.is_cuda and sub_bus.device == dev and sub_bus.dim() == 2 and sub_bus.shape[0] == B
                    and sub_bus.shape[1] >= self.max_sub_size and sub_bus.dtype in (torch.int8,) + ints):
                raise ValueError(f"sub_bus must be an int8 / int32 / int64 CUDA tensor of shape ({B}, >= {self.max_sub_size}) on {dev}")
            sb = sub_bus if sub_bus.dtype == torch.int8 else sub_bus.clamp(-128, 127).to(torch.int8)
            if sb.stride(1) != 1:
                sb = sb.contiguous()
            keep.append(sb)
            sbus, cols, stride = sb.data_ptr(), sb.shape[1], sb.stride(0)
        if line_id is not None:
            lid = ids(line_id, "line_id")
            lst = ids(line_status, "line_status")
        aid = ids(action_id, "action_id") if action_id is not None else 0
        if raise_alert is not None:
            if self._alerts is None:
                raise ValueError("raise_alert without enable_alerts()")
            _check_tensor(raise_alert, "raise_alert", (B, self._alerts.n), (torch.bool, torch.uint8), dev)
        if raise_alarm is not None:
            if self._alarms is None:
                raise ValueError("raise_alarm without enable_alarms()")
            _check_tensor(raise_alarm, "raise_alarm", (B, self._alarms.n), (torch.bool, torch.uint8), dev)
        if self._authority != "device":
            self._to_device()
        if self._alerts is not None:                      # (on torch's stream: ordered before the engine's launches below)
            if raise_alert is None:
                d["alert_raise"].zero_()
            else:
                d["alert_raise"].copy_(raise_alert != 0)
        if self._alarms is not None:
            if raise_alarm is None:
                d["alarm_raise"].zero_()
            else:
                d["alarm_raise"].copy_(raise_alarm != 0)
        if use_vec:                                       # (device to device, on torch's stream like the alert buffers)
            for (x, _, _, _), key in zip(vec, ("act_set_bus", "act_change_bus", "act_set_status", "act_change_status")):
                if x is None:
                    d[key].zero_()
                else:
                    d[key].copy_(x)
        cur, eng = self._streams()
        eng.wait_stream(cur)
        try:
            if aid:
                self.engine.env_step_ids(aid, from_reset=from_reset, is_dc=self.is_dc, max_iter=self.max_iter, tol_mva=self.tol_mva,
                                         tight_cap=self.tight_cap, stamp=self.n_steps + 1)
            elif use_vec:
                self.engine.env_step_act(from_reset=from_reset, is_dc=self.is_dc, max_iter=self.max_iter, tol_mva=self.tol_mva,
                                         tight_cap=self.tight_cap, stamp=self.n_steps + 1)
            else:
                self.engine.env_step(sid, sbus, stride, cols, lid, lst, from_reset=from_reset, is_dc=self.is_dc, max_iter=self.max_iter,
                                     tol_mva=self.tol_mva, tight_cap=self.tight_cap, stamp=self.n_steps + 1)
        except RuntimeError as e:
            if "(-1)" in str(e):                          # B200PF_E_ARG: an action out of range, nothing was written
                raise ValueError(str(e)) from None
            raise
        cur.wait_stream(eng)
        self.n_steps += 1
        self._n_dev_steps = getattr(self, "_n_dev_steps", 0) + 1     # (as step_device counts them: simulate_forecast reads it)
        st = self.engine.env_stats()
        self.n_illegal += st["n_illegal"] - self._illegal_seen
        self._illegal_seen = st["n_illegal"]
        if self.tight_cap:
            self.nb_cap = st["nb_cap"]
        info = {"status": d["status"], "iters": d["iters"], "newly_done": d["newly_done"], "is_illegal": d["is_illegal"],
                "disc_lines": d["disc"] if self.protections else None}
        if use_vec or aid:
            info["is_ambiguous"] = d["is_ambiguous"]
        if self._opp is not None:
            info["opponent_attack_line"] = d["opp_lines"] if self._opp.multi else d["opp_line"]
            info["opponent_attack_duration"] = d["opp_dur"]
        if self._alerts is not None and self._alerts.reward:
            info["rewards"] = {"alert": d["alert_reward"]}
        if self._alarms is not None:
            info["is_alarm_illegal"] = d["alarm_illegal"]
            if self._alarms.reward:
                info["rewards"] = {"alarm": d["alarm_reward"]}
        return d["rho"], d["done"], info

    def _reset_tensors(self, mask, rows=None):
        import torch
        d = self._tensor_state()
        dev, B = d["device"], self.batch
        _check_tensor(mask, "mask", (B,), (torch.bool,), dev)
        m = mask.contiguous()
        r = None
        if rows is not None:
            _check_tensor(rows, "rows", (B,), (torch.int32, torch.int64), dev)
            r = torch.remainder(rows, self.chron.shape[1]).to(torch.int32).contiguous()
        if self._authority != "device":
            self._to_device()
        cur, eng = self._streams()
        eng.wait_stream(cur)
        self.engine.env_reset(m.data_ptr(), 0 if r is None else r.data_ptr())
        cur.wait_stream(eng)
        m.record_stream(eng)                              # (the mask / rows may be freed before the engine's stream read them)
        if r is not None:
            r.record_stream(eng)

    def reset_step(self):
        """the solve ``env.reset()`` performs on the first row (no soft-overflow counting, no cooldown from actions)"""
        return self.step(from_reset=True)


def _is_cuda_tensor(x) -> bool:
    try:
        import torch
    except ImportError:                                   # pragma: no cover
        return False
    return torch.is_tensor(x) and x.is_cuda


def _check_tensor(x, name, shape, dtypes, device):
    import torch
    if not (torch.is_tensor(x) and x.is_cuda and x.device == device and tuple(x.shape) == tuple(shape) and x.dtype in dtypes):
        raise ValueError(f"{name} must be a CUDA tensor of shape {tuple(shape)} and dtype {' / '.join(str(t) for t in dtypes)} on {device}")


class _DeviceArray:
    """``__cuda_array_interface__`` of device memory the engine owns (zero-copy torch views)"""

    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = dict(shape=tuple(shape), typestr=typestr, data=(int(ptr), False), version=2, strides=None)


def _device_view(ptr, shape, typestr, device):
    import torch
    return torch.as_tensor(_DeviceArray(ptr, shape, typestr), device=device)


def random_substation_actions(env: BatchedEnv, rng: np.random.Generator):
    """BASELINE.json configs[2] / SURVEY.md 8(d) config 3: every instance draws one substation and a uniformly random busbar
    in {1, 2} for each of its elements (``MAX_SUB_CHANGED = 1``).  -> (sub_id [B], sub_bus [B, max_sub_size])"""
    B = env.batch
    sub = rng.integers(0, env.gm.n_sub, B)
    bus = rng.integers(1, 3, (B, env.max_sub_size)).astype(np.int8)
    bus[np.arange(env.max_sub_size)[None, :] >= env.sub_size[sub][:, None]] = 0
    return sub, bus
