"""Grid features no bundled grid has, and topologies at the size limits of the solver kernels: the helpers the GPU file
(test_kernel_limits_gpu.py) builds its cases with, checked on the host.

* ``psh(gm, deg)``: phase-shifting transformers.  Every bundled grid has ``shift_degree = 0`` on all its transformers, so
  the shifts are made by rotating the admittances of the transformer rows in place; the first test shows that this is
  what a grid file with those ``shift_degree`` values gives.
* ``variant(key)``: the grids of the limit tests — shifts, three busbars per substation, and case14 with a line inside a
  substation and a pair of parallel lines (``case14_odd`` of test_block_ybus_cpu.py), alone and combined.
* ``heavy_splits(gm, n, seed)``: topologies with every substation split at random over its busbars, still connected.
* ``BOUNDARY``: sets of states with exactly the active-bus counts where the pivoting path changes its kernel class.

Checked here: the numpy oracle agrees with the C oracle on these grids (the GPU tests trust the C oracle on features no
``res_*`` table of the reference covers), and the host builds of the planned kernels agree with the C oracle on them."""
import os

import numpy as np
import pytest

from conftest import env_grid

from grid2op_b200.engine import grid_max_active_buses
from grid2op_b200.gridmodel import GridModel
from oracle.c_oracle import COracle
from test_block_ybus_cpu import _grid
from test_c_oracle import random_cases
from test_sparse_plan_cpu import compare

GOLD = os.path.join(os.path.dirname(__file__), "golden")


# ---- grid variants ---------------------------------------------------------------------------------------------------
def shifts(gm, deg=15.0):
    """one shift per transformer: magnitudes from 3 to deg degrees, alternating signs"""
    n = gm.n_trafo
    return np.where(np.arange(n) % 2 == 1, 1.0, -1.0) * np.linspace(3.0, deg, n)


def psh(gm, deg):
    """Phase shift of deg[k] degrees on transformer k (the last n_trafo rows of the branch tables), in place.  With
    tap = ratio e^{j phi} (GridModel): y_ft = -y_s / conj(tap) turns by e^{j phi}, y_tf = -y_s / tap by e^{-j phi}, y_ff and
    y_tt keep their values, and the DC model gets line_pshift = -b_dc phi.  The grid must have no shift yet."""
    rows = np.arange(gm.n_line - gm.n_trafo, gm.n_line)
    phi = np.deg2rad(np.broadcast_to(np.asarray(deg, dtype=np.float64), rows.shape))
    assert not np.asarray(gm.line_pshift).any()
    y = np.array(gm.line_y, dtype=np.float64).reshape(gm.n_line, 8)
    for k, sign in ((1, 1.0), (2, -1.0)):                  # (y_ff, y_ft, y_tf, y_tt) as (re, im) pairs
        c = (y[rows, 2 * k] + 1j * y[rows, 2 * k + 1]) * np.exp(1j * sign * phi)
        y[rows, 2 * k], y[rows, 2 * k + 1] = c.real, c.imag
    gm.line_y = y
    p = np.array(gm.line_pshift, dtype=np.float64)
    p[rows] = -np.asarray(gm.line_bdc, dtype=np.float64)[rows] * phi
    gm.line_pshift = p
    return gm


def variant(key):
    """'<grid>[+b3][+psh]': the grid (golden model, or the grid file for three busbars per substation), "case14_odd" for
    case14 with a line inside a substation and a pair of parallel lines; +b3: three busbars; +psh: shifts(gm)"""
    grid, *feat = key.split("+")
    if "b3" in feat:
        path = env_grid(grid)
        if path is None:
            pytest.skip("reference grid files not available")
        gm = GridModel(path, n_busbar=3)
    else:
        gm = _grid(grid)
    if "psh" in feat:
        psh(gm, shifts(gm))
    return gm


# ---- topologies ------------------------------------------------------------------------------------------------------
def _sub_of_input(gm):
    """substation of every topology input: elements, shunts, reference units"""
    s = np.full(gm.n_topo_in, -1, dtype=np.int64)
    s[gm.line_or_pos] = gm.line_or_sub
    s[gm.line_ex_pos] = gm.line_ex_sub
    s[gm.gen_pos] = gm.gen_sub
    s[gm.load_pos] = gm.load_sub
    if gm.n_storage:
        s[gm.storage_pos] = gm.storage_sub
    s[gm.dim_topo:gm.dim_topo + gm.n_shunt] = gm.shunt_sub
    s[gm.dim_topo + gm.n_shunt:] = gm.hidden_sub
    return s


def _buses(gm, tv, sub_of):
    """(active buses, whether every active bus reaches every other one over in-service lines)"""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    slot = sub_of * gm.n_busbar + tv.astype(np.int64) - 1
    active = np.unique(slot[tv > 0])
    lo, le = gm.line_or_pos, gm.line_ex_pos
    on = (tv[lo] > 0) & (tv[le] > 0)
    m = coo_matrix((np.ones(int(on.sum())), (slot[lo][on], slot[le][on])), shape=(gm.n_slot, gm.n_slot))
    lab = connected_components(m, directed=False)[1]
    return len(active), len(np.unique(lab[active])) == 1


def heavy_splits(gm, n, seed, target=None, tries=6):
    """Heavy connected splits: the substations in random order, every element of one on a random busbar 1..n_busbar.  A draw
    is kept only if the active buses still reach each other over in-service lines; after `tries` draws the substation keeps
    its busbars.  target: a draw that would give more active buses is not kept, and the instance is done when it has
    exactly that many."""
    rng = np.random.default_rng(seed)
    sub_of = _sub_of_input(gm)
    topo = np.tile(gm.default_topo(), (n, 1))
    for i in range(n):
        tv = topo[i]
        nb = _buses(gm, tv, sub_of)[0]
        for s in rng.permutation(gm.n_sub):
            if target is not None and nb == target:
                break
            pos = np.flatnonzero((sub_of == s) & (tv > 0))
            for _ in range(tries):
                t2 = tv.copy()
                t2[pos] = rng.integers(1, gm.n_busbar + 1, len(pos))
                nb2, ok = _buses(gm, t2, sub_of)
                if ok and (target is None or nb2 <= target):
                    tv[:], nb = t2, nb2
                    break
    return topo


# boundary sets: variant -> (exact active-bus counts, instances per count, seed).  17 / 18: the warp-per-instance kernel takes
# up to 17 buses (and only grids with <= 32 bus slots); 128 / 129: the generic kernel's last threads-per-instance step.
BOUNDARY = {"l2rpn_case14_sandbox+psh": ((17, 18), 12, 97), "l2rpn_case14_sandbox+b3+psh": ((17, 18), 12, 101),
            "l2rpn_wcci_2022_dev+b3+psh": ((128, 129), 6, 103)}


def boundary_states(gm, key):
    """BOUNDARY[key] states at default injections: {count: topologies}"""
    counts, n, seed = BOUNDARY[key]
    return {c: heavy_splits(gm, n, seed + c, target=c) for c in counts}


def solved(gm, topo, max_iters=6):
    """the instances the oracle solves at default injections in at most max_iters Newton iterations (a state that needs more
    lies close to voltage collapse, where an fp32 and an fp64 Jacobian may end on different sides of the iteration limit:
    test_redo_gpu.py), as (topo, inj, the oracle's AC results)"""
    inj = np.tile(gm.default_inj(), (len(topo), 1))
    ref, st, it, _ = COracle(gm).run(topo, inj)
    k = (st == 0) & (it <= max_iters)
    return topo[k], inj[k], (ref[k], st[k], it[k])


# ---- 1. the rotation is what a grid file with shift_degree gives -----------------------------------------------------
def _shifted_file(tmp_path, name, n_busbar=2):
    """(a copy of the grid file with shifts(gm) as the transformers' shift_degree, its GridModel)"""
    from grid2op_b200.ppjson import update_pp_json
    path = env_grid(name)
    if path is None:
        pytest.skip("reference grid files not available")
    gm = GridModel(path, n_busbar=n_busbar)
    dst = str(tmp_path / f"{name}_psh.json")
    update_pp_json(path, dst, {"trafo": {"shift_degree": shifts(gm)}})
    return path, GridModel(dst, n_busbar=n_busbar)


@pytest.mark.parametrize("name", ["l2rpn_case14_sandbox", "l2rpn_neurips_2020_track1", "l2rpn_wcci_2022_dev"])
def test_rotation_equals_the_grid_file_with_shift_degree(tmp_path, name):
    path, gf = _shifted_file(tmp_path, name)
    gm = GridModel(path)
    assert gm.n_trafo >= 4 and not gm.line_pshift.any()
    psh(gm, shifts(gm))
    assert gf.line_pshift[-gm.n_trafo:].all() and not gf.line_pshift[:-gm.n_trafo].any()
    scale = np.abs(gf.line_y).max()
    assert np.max(np.abs(gm.line_y - gf.line_y)) <= 1e-13 * scale, np.max(np.abs(gm.line_y - gf.line_y)) / scale
    assert np.allclose(gm.line_pshift, gf.line_pshift, rtol=1e-13, atol=0.0)
    assert np.array_equal(gm.line_bdc, gf.line_bdc)
    # the mutual admittances of a shifted branch differ (y_ft != y_tf), and only there
    y = gf.line_y.reshape(-1, 8)
    asym = np.abs(y[:, 2:4] - y[:, 4:6]).max(axis=1) > 1e-9 * np.abs(y[:, 2:4]).max(axis=1)
    assert np.array_equal(asym, gf.line_pshift != 0)


# ---- 2. the numpy oracle agrees with the C oracle on the variants ----------------------------------------------------
@pytest.mark.parametrize("name,n_busbar", [("l2rpn_case14_sandbox", 2), ("l2rpn_case14_sandbox", 3), ("l2rpn_neurips_2020_track1", 3)])
@pytest.mark.parametrize("dc", [False, True])
def test_numpy_oracle_matches_c_oracle_on_shifts_and_three_busbars(tmp_path, name, n_busbar, dc):
    """the numpy oracle reads the edited grid file; the C oracle gets the in-place rotation of the GPU tests"""
    from oracle_engine import OracleEngine
    path, gf = _shifted_file(tmp_path, name, n_busbar)
    gm = psh(GridModel(path, n_busbar=n_busbar), shifts(gf))
    t1, i1 = random_cases(gm, 16, seed=7)
    t2 = heavy_splits(gm, 8, seed=9)
    topo, inj = np.concatenate([t1, t2]), np.concatenate([i1, np.tile(gm.default_inj(), (len(t2), 1))])
    assert (topo == n_busbar).any()
    o1, s1, i1, _ = OracleEngine(gf).run(topo, inj, is_dc=dc)
    o2, s2, i2, _ = COracle(gm, nthreads=2).run(topo, inj, is_dc=dc)
    assert (s1 == 0).sum() >= 8
    assert np.array_equal(s1 == 0, s2 == 0), (s1, s2)
    ok = s1 == 0
    assert np.max(np.abs(o1[ok] - o2[ok]) / (1.0 + np.abs(o1[ok]))) <= 2e-5      # (test_c_oracle.py)
    if not dc:
        assert np.array_equal(i1[ok], i2[ok])


# ---- 3. the host builds of the planned kernels on the variants --------------------------------------------------------
@pytest.mark.parametrize("key,n", [("l2rpn_case14_sandbox+psh", 48), ("case14_odd+psh", 48), ("l2rpn_case14_sandbox+b3+psh", 48),
                                   ("l2rpn_neurips_2020_track1+b3+psh", 12)])
@pytest.mark.parametrize("dc", [False, True])
def test_host_builds_of_the_planned_kernels_vs_c_oracle(key, n, dc):
    from sparse_emu import BlockEmu, SparseEmu
    gm = variant(key)
    t1, i1 = random_cases(gm, n, seed=13)
    t2 = heavy_splits(gm, n, seed=15)
    topo, inj = np.concatenate([t1, t2]), np.concatenate([i1, np.tile(gm.default_inj(), (n, 1))])
    ref, rstatus, riters, _ = COracle(gm).run(topo, inj, is_dc=dc)
    assert (rstatus == 0).sum() >= n // 2 and (rstatus != 0).any()
    emus = [SparseEmu(gm), BlockEmu(gm, 8, 1)] + ([BlockEmu(gm, 32, 1)] if gm.n_line > 32 else [])
    for emu in emus:
        out, status, iters, _ = emu.run(topo, inj, is_dc=dc)
        assert np.array_equal(status, rstatus), type(emu).__name__
        ok = status == 0
        assert np.isnan(out[~ok]).all()
        compare(gm, out, ref, ok)
        if not dc:
            d = iters[ok] - riters[ok]
            assert d.min() >= 0 and d.max() <= 1, (type(emu).__name__, d.min(), d.max())


# ---- 4. the generator reaches the bus counts the GPU tests rely on ----------------------------------------------------
@pytest.mark.parametrize("key,lo,hi", [("l2rpn_case14_sandbox+psh", 19, 28), ("l2rpn_case14_sandbox+b3+psh", 19, 42),
                                       ("l2rpn_neurips_2020_track1+b3+psh", 52, 108)])
def test_heavy_splits_reach_their_bus_counts(key, lo, hi):
    """connected, and well above the file's bus count: case14 about 20 buses, track1 about 56 to 60"""
    gm = variant(key)
    topo = heavy_splits(gm, 24, seed=5)
    sub_of = _sub_of_input(gm)
    assert all(_buses(gm, t, sub_of)[1] for t in topo)
    nb = grid_max_active_buses(gm, topo)[1]
    assert nb.min() >= lo and nb.max() <= hi, (nb.min(), nb.max())
    assert np.median(nb) >= lo + 1, np.median(nb)


@pytest.mark.parametrize("key", sorted(BOUNDARY))
def test_boundary_sets_have_exactly_their_bus_counts(key):
    gm = variant(key)
    sets = boundary_states(gm, key)
    sub_of = _sub_of_input(gm)
    for c, topo in sets.items():
        assert np.array_equal(grid_max_active_buses(gm, topo)[1], np.full(len(topo), c)), c
        assert all(_buses(gm, t, sub_of)[1] for t in topo)
        assert len(solved(gm, topo)[0]) >= 2, c
