"""A discrete action table for :class:`grid2op_b200.batched_env.BatchedEnv`: the list of topology actions an RL agent indexes with
one integer per environment (grid2op's ``IdToAct`` converter, grid2op/Converter/IdToAct.py, or a filtered list saved with
``IdToAct.save``).  Each row holds grid2op's native topology action in the layout of BatchedEnv's vector action; the environment
validates the table once, when it is bound (:meth:`BatchedEnv.set_action_table`), and each step reads only the row of each id.
"""
from __future__ import annotations

import numpy as np

from .gridmodel import GridModel

__all__ = ["ActionTable"]


class ActionTable:
    """``set_bus`` int8 [n, dim_topo] (0 leave, -1 disconnect a line end, 1..n_busbar), ``change_bus`` bool [n, dim_topo] (two
    busbars per substation only), ``set_line_status`` int8 [n, n_line] in {-1, 0, 1}, ``change_line_status`` bool [n, n_line].  Any
    subset may be given; a missing one is zeros.  A value out of range, ``set_bus = -1`` on a load, generator or storage unit
    (detachment), a wrong shape or dtype raise ValueError.  The arrays are read-only once the table is built."""

    def __init__(self, gm: GridModel, set_bus=None, change_bus=None, set_line_status=None, change_line_status=None):
        self.dim_topo, self.n_line, self.n_busbar = int(gm.dim_topo), int(gm.n_line), int(gm.n_busbar)
        given = [x for x in (set_bus, change_bus, set_line_status, change_line_status) if x is not None]
        if not given:
            raise ValueError("an action table needs at least one of set_bus, change_bus, set_line_status, change_line_status")
        n = len(np.asarray(given[0]))
        out = []
        for x, name, w, kinds in ((set_bus, "set_bus", self.dim_topo, "iu"), (change_bus, "change_bus", self.dim_topo, "b"),
                                  (set_line_status, "set_line_status", self.n_line, "iu"),
                                  (change_line_status, "change_line_status", self.n_line, "b")):
            dt = bool if kinds == "b" else np.int8
            if x is None:
                out.append(np.zeros((n, w), dtype=dt))
                continue
            x = np.asarray(x)
            if x.shape != (n, w) or x.dtype.kind not in kinds:
                raise ValueError(f"{name} must be a {'bool' if kinds == 'b' else 'int'} array of shape {(n, w)}")
            if kinds != "b" and ((x < -1) | (x > 127)).any():           # (before the narrowing to int8)
                raise ValueError(f"{name} out of range")
            out.append(np.ascontiguousarray(x, dtype=dt))
        sb, cb, ss, cs = out
        line_end = np.zeros(self.dim_topo, dtype=bool)
        line_end[np.asarray(gm.line_or_pos)] = True
        line_end[np.asarray(gm.line_ex_pos)] = True
        bad = np.flatnonzero(((sb < -1) | (sb > self.n_busbar)).any(axis=1))
        if len(bad):
            raise ValueError(f"set_bus outside [-1, {self.n_busbar}] in row {int(bad[0])}")
        bad = np.flatnonzero(((sb == -1) & ~line_end[None, :]).any(axis=1))
        if len(bad):
            raise ValueError(f"set_bus = -1 on a load, generator or storage unit in row {int(bad[0])} (detachment is not supported)")
        if cb.any() and self.n_busbar != 2:
            raise ValueError("change_bus needs two busbars per substation")
        bad = np.flatnonzero(((ss < -1) | (ss > 1)).any(axis=1))
        if len(bad):
            raise ValueError(f"set_line_status outside {{-1, 0, 1}} in row {int(bad[0])}")
        for a in out:
            a.setflags(write=False)
        self.set_bus, self.change_bus, self.set_line_status, self.change_line_status = sb, cb, ss, cs
        self.n = n

    def __len__(self) -> int:
        return self.n

    def matches(self, gm: GridModel) -> bool:
        """the table was built for a grid of these dimensions"""
        return (self.dim_topo, self.n_line, self.n_busbar) == (int(gm.dim_topo), int(gm.n_line), int(gm.n_busbar))

    # ---- the table of IdToAct.init_converter ---------------------------------------------------------------------------------
    @classmethod
    def unitary(cls, gm: GridModel, set_line_status: bool = True, change_line_status: bool = True, set_topo_vect: bool = True,
                change_bus_vect: bool = True) -> "ActionTable":
        """The topology part of ``IdToAct(action_space).init_converter(redispatch=False, curtail=False, storage=False)``, in its
        order, with a flag per kind of action (set them as the environment's action class has them):

        0. do nothing;
        1. ``set_line_status``: every line disconnected, then every line reconnected with its extremity on busbar ``b1`` and its
           origin on ``b2``, for ``(b1, b2)`` over the pairs of busbars in lexicographic order (outer loop) and the lines (inner);
        2. ``change_line_status``: one action per line;
        3. ``set_topo_vect``: per substation, every assignment of its elements (topology-vector order) to busbars with the first
           on busbar 1, in lexicographic order, kept when the busbars are numbered in their order of first use (up to the
           second-to-last busbar) and when every busbar used carries a line end; a substation with fewer than two such
           assignments adds none;
        4. ``change_bus_vect``: per substation, every subset of its elements that leaves the first one alone, except the empty
           one, in lexicographic order (a subset and its complement have the same effect).  Needs two busbars per substation
           (ValueError otherwise)."""
        if change_bus_vect and gm.n_busbar != 2:
            raise ValueError("change_bus actions need exactly two busbars per substation")
        nt, nl, nb = int(gm.dim_topo), int(gm.n_line), int(gm.n_busbar)
        sub_info = np.asarray(gm.sub_info, dtype=np.int64)
        start = np.concatenate([[0], np.cumsum(sub_info)[:-1]])
        # local index (within its substation) of each line end, per substation
        line_local = [[] for _ in range(len(sub_info))]
        for s, p in zip(np.asarray(gm.line_or_sub), np.asarray(gm.line_or_to_sub_pos)):
            line_local[int(s)].append(int(p))
        for s, p in zip(np.asarray(gm.line_ex_sub), np.asarray(gm.line_ex_to_sub_pos)):
            line_local[int(s)].append(int(p))
        lor, lex = np.asarray(gm.line_or_pos, dtype=np.int64), np.asarray(gm.line_ex_pos, dtype=np.int64)
        sb_parts, cb_parts, ss_parts, cs_parts = [np.zeros((1, nt), np.int8)], [np.zeros((1, nt), bool)], [np.zeros((1, nl), np.int8)], \
            [np.zeros((1, nl), bool)]

        def add(sb=None, cb=None, ss=None, cs=None, n=0):
            sb_parts.append(np.zeros((n, nt), np.int8) if sb is None else sb)
            cb_parts.append(np.zeros((n, nt), bool) if cb is None else cb)
            ss_parts.append(np.zeros((n, nl), np.int8) if ss is None else ss)
            cs_parts.append(np.zeros((n, nl), bool) if cs is None else cs)

        eye = np.arange(nl)
        if set_line_status:
            ss = np.zeros((nl, nl), np.int8); ss[eye, eye] = -1
            add(ss=ss, n=nl)
            for b_ex in range(1, nb + 1):
                for b_or in range(1, nb + 1):
                    ss = np.zeros((nl, nl), np.int8); ss[eye, eye] = 1
                    sb = np.zeros((nl, nt), np.int8); sb[eye, lor] = b_or; sb[eye, lex] = b_ex
                    add(sb=sb, ss=ss, n=nl)
        if change_line_status:
            cs = np.zeros((nl, nl), bool); cs[eye, eye] = True
            add(cs=cs, n=nl)
        if set_topo_vect and nb > 1:
            for s, k in enumerate(sub_info):
                tup = _assignments(nb, int(k))
                ok = _numbered_in_order(tup, nb)
                lines = tup[:, line_local[s]]
                used = np.stack([(lines == b).any(axis=1) for b in range(1, nb + 1)], axis=1).sum(axis=1)
                ok &= used == tup.max(axis=1)
                tup = tup[ok]
                if len(tup) < 2:
                    continue
                sb = np.zeros((len(tup), nt), np.int8)
                sb[:, start[s]:start[s] + k] = tup
                add(sb=sb, n=len(tup))
        if change_bus_vect:
            for s, k in enumerate(sub_info):
                k = int(k)
                if k < 2:
                    continue
                tup = _assignments(2, k) - 1                         # the subsets with the first element left alone, in order
                tup = tup[1:].astype(bool)                           # (without the empty one)
                cb = np.zeros((len(tup), nt), bool)
                cb[:, start[s]:start[s] + k] = tup
                add(cb=cb, n=len(tup))
        return cls(gm, np.concatenate(sb_parts), np.concatenate(cb_parts), np.concatenate(ss_parts), np.concatenate(cs_parts))

    # ---- a list of grid2op actions -------------------------------------------------------------------------------------------
    @classmethod
    def from_actions(cls, gm: GridModel, actions) -> "ActionTable":
        """The table of a list of grid2op action objects, ``converter.all_actions`` of an ``IdToAct`` say (restored from a saved
        ``.npy`` or not): their ``set_bus``, ``change_bus``, ``line_set_status`` and ``line_change_status``.  ValueError for an
        action that also modifies injections, voltages, redispatching, storage or curtailment (``get_types()``), that raises an
        alarm or an alert, that detaches an element, or whose vectors do not have this grid's dimensions."""
        actions = list(actions)
        if not actions:
            raise ValueError("no actions")
        sb, cb, ss, cs = [], [], [], []
        for k, a in enumerate(actions):
            injection, voltage, _, _, redispatching, storage, curtailment = a.get_types()[:7]
            kinds = [nm for nm, on in (("injection", injection), ("voltage", voltage), ("redispatching", redispatching),
                                       ("storage", storage), ("curtailment", curtailment)) if on]
            if kinds:
                raise ValueError(f"action {k} modifies {', '.join(kinds)}: only topology actions go in an action table")
            for attr in ("raise_alarm", "raise_alert"):
                v = getattr(type(a), "dim_alarms" if attr == "raise_alarm" else "dim_alerts", 0)
                if v and np.asarray(getattr(a, attr)).any():
                    raise ValueError(f"action {k} raises an {attr[6:]}: only topology actions go in an action table")
            x = [np.asarray(a.set_bus), np.asarray(a.change_bus), np.asarray(a.line_set_status), np.asarray(a.line_change_status)]
            if [len(v) for v in x] != [gm.dim_topo, gm.dim_topo, gm.n_line, gm.n_line]:
                raise ValueError(f"action {k} is for another grid (dim_topo {len(x[0])}, n_line {len(x[2])})")
            for lst, v in zip((sb, cb, ss, cs), x):
                lst.append(v)
        return cls(gm, np.stack(sb).astype(np.int64), np.stack(cb).astype(bool), np.stack(ss).astype(np.int64), np.stack(cs).astype(bool))


def _assignments(nb: int, k: int) -> np.ndarray:
    """int [nb ** (k - 1), k]: the first element on busbar 1, the others over 1..nb, in lexicographic order"""
    m = k - 1
    idx = np.arange(nb ** m, dtype=np.int64)
    digits = (idx[:, None] // (nb ** np.arange(m - 1, -1, -1, dtype=np.int64))[None, :]) % nb + 1
    return np.concatenate([np.ones((len(idx), 1), np.int64), digits], axis=1)


def _numbered_in_order(tup: np.ndarray, nb: int) -> np.ndarray:
    """bool [n]: each busbar below ``nb - 1`` appears before the next one (a busbar may be new only when it is the highest seen so
    far plus one); once the highest busbar seen reaches ``nb - 1`` anything may follow"""
    seen = np.maximum.accumulate(tup, axis=1)
    prev = seen[:, :-1]
    ok = (prev >= nb - 1) | (tup[:, 1:] <= prev + 1)
    return ok.all(axis=1)
