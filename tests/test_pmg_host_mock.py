"""Host logic of p-multigrid on the CPU.

* The solver options (defaults, nested dicts, refusals by name), the refusals of mg.PMG and mg.PTransfer, and the DQ
  message of solve, which p-multigrid leaves unchanged.
* Against PMGEngine, a mock engine that computes the transfers and fdb_vec_chebyshev in NumPy and records every
  engine call: the calls of one PMGPC and one P1PC cycle at p = 2 and 3, the mock's transfers against the oracle, and
  the outer iterations that bound tests/test_pmg_gpu.py::test_poisson_iterations.
* solve() with pc_type none, jacobi and mg makes the engine calls it made on the parent commit (SOLVE_CALLS)."""
import numpy as np
import pytest

import _mock_engine as me
import _pmg_oracle as po
from firedrake_b200 import _lib, mg
from firedrake_b200.assemble import DirichletBC, Form, FunctionSpace, assemble, mass, pmg_options, solve
from firedrake_b200.utility_meshes import ExtrudedHexMesh

PMG = {"pc_type": "python", "pc_python_type": "firedrake.PMGPC"}
P1 = {"pc_type": "python", "pc_python_type": "firedrake.P1PC"}


def test_defaults_and_kinds():
    o = pmg_options(PMG)
    assert o["halve"] and o["pmg_mg_coarse_degree"] == 1
    assert (o["pmg_mg_levels_ksp_type"], o["pmg_mg_levels_ksp_max_it"], o["pmg_mg_levels_pc_type"]) == \
        ("chebyshev", 2, "jacobi")
    assert o["pmg_mg_levels_ksp_chebyshev_esteig"] == "0,0.1,0,1.1"
    assert (o["pmg_mg_coarse_ksp_type"], o["pmg_mg_coarse_pc_type"]) == ("cg", "jacobi")
    assert not pmg_options({"pc_python_type": "firedrake.P1PC"})["halve"]
    with pytest.raises(NotImplementedError, match="pc_python_type 'firedrake.ASMStarPC'"):
        pmg_options({"pc_python_type": "firedrake.ASMStarPC"})


def test_nested_dicts_are_flattened():
    o = pmg_options(dict(PMG, pmg_mg_levels={"ksp_type": "richardson", "ksp_max_it": 3},
                         pmg_mg_coarse={"ksp_type": "preonly", "pc_type": "mg"}, pmg_mg_coarse_degree=2))
    assert (o["pmg_mg_levels_ksp_type"], o["pmg_mg_levels_ksp_max_it"]) == ("richardson", 3)
    assert (o["pmg_mg_coarse_ksp_type"], o["pmg_mg_coarse_pc_type"], o["pmg_mg_coarse_degree"]) == ("preonly", "mg", 2)


def test_unknown_and_unsupported_options_are_refused():
    with pytest.raises(NotImplementedError, match="pmg_mg_levels_pc_python_type"):
        pmg_options(dict(PMG, pmg_mg_levels={"pc_python_type": "x"}))
    with pytest.raises(NotImplementedError, match="pmg_foo"):
        pmg_options(dict(PMG, pmg_foo=1))
    with pytest.raises(NotImplementedError, match="pmg_mg_levels_pc_type 'sor'"):
        pmg_options(dict(PMG, pmg_mg_levels_pc_type="sor"))


def _make(W, k=None):
    return Form(W)


def test_pmg_refusals():
    mesh = ExtrudedHexMesh(3, 3, 3)
    with pytest.raises(ValueError, match="fine degree 1 has nothing to coarsen"):
        mg.PMG(FunctionSpace(mesh, 1), _make)
    for p in (4, 5):
        with pytest.raises(NotImplementedError, match=f"fine degree {p}"):
            mg.PMG(FunctionSpace(mesh, p), _make)
    with pytest.raises(NotImplementedError, match="partitioned"):
        mg.PMG(FunctionSpace(mesh, 2), _make, allreduce=lambda v: v)
    with pytest.raises(ValueError, match="needs a mesh hierarchy whose finest mesh is V's mesh"):
        mg.PMG(FunctionSpace(mesh, 3), _make, coarse_ksp="preonly", coarse_pc="mg")
    h = mg.MeshHierarchy(2, 2, 2, 1)                         # finest 4^3: not this 3^3 mesh
    with pytest.raises(ValueError, match="needs a mesh hierarchy whose finest mesh is V's mesh"):
        mg.PMG(FunctionSpace(mesh, 3), _make, coarse_ksp="preonly", coarse_pc="mg", hierarchy=h)
    # an equal mesh that is another object: the levels must share the mesh itself
    with pytest.raises(ValueError, match="needs a mesh hierarchy whose finest mesh is V's mesh"):
        mg.PMG(FunctionSpace(ExtrudedHexMesh(4, 4, 4), 3), _make, coarse_ksp="preonly", coarse_pc="mg", hierarchy=h)
    with pytest.raises(ValueError, match="steps must be at least 1"):
        mg.jacobi_lanczos_bounds(None, None, None, steps=0)
    with pytest.raises(NotImplementedError, match="coarse solve ksp_type 'preonly' with pc_type 'jacobi'"):
        mg.PMG(FunctionSpace(mesh, 3), _make, coarse_ksp="preonly", coarse_pc="jacobi")
    with pytest.raises(NotImplementedError, match="level smoother 'sor'"):
        mg.PMG(FunctionSpace(mesh, 3), _make, smoother="sor")
    with pytest.raises(NotImplementedError, match="no DQ p-multigrid"):
        mg.PMG(FunctionSpace(mesh, 2, family="DQ"), _make)
    with pytest.raises(ValueError, match="same mesh"):
        mg.PTransfer(FunctionSpace(mesh, 1), FunctionSpace(ExtrudedHexMesh(3, 3, 3), 2))


def test_dq_message_unchanged():
    V = FunctionSpace(ExtrudedHexMesh(2, 2, 2), 2, family="DQ")
    with pytest.raises(NotImplementedError, match=r"pc_type 'python' on a DQ space: 'none' or 'jacobi' \(there is no "
                                                  r"DQ multigrid\)"):
        solve(Form(V), V.dat(), V.dat(np.zeros(V.node_count)), solver_parameters=PMG)


# ---------------------------------------------------------------------------------------------------------------
# A mock engine that computes the p-multigrid kernels in NumPy (the transfers and fdb_vec_chebyshev), the Helmholtz
# family through the oracle (tests/_mock_engine.py) and the generated wrappers through their host build, and records
# every kernel call and vector operation in order.

_TRANSFERS = {_lib.FORM_P_PROLONG: "p_prolong", _lib.FORM_P_RESTRICT: "p_restrict", _lib.FORM_P_INJECT: "p_inject"}
_RECORDED = ("fdb_vec_axpy", "fdb_vec_aypx", "fdb_vec_scale", "fdb_vec_dot", "fdb_vec_pointwise_mult",
             "fdb_dat_zero_nodes", "fdb_dat_set_nodes", "fdb_dat_set_nodes_scalar", "fdb_memset", "fdb_memcpy_d2d")


def _kron3(T):
    return np.kron(np.kron(T, T), T)


class PMGEngine(me.MockEngine):
    """The mock engine with the p-multigrid kernels, recording ``trace``: ("helmholtz", degree, "action" | "diagonal"),
    ("jit", name), (transfer form, p, q) per kernel call and (name, n) per vector operation."""

    def __init__(self, oracle, compute=True):
        super().__init__(oracle)
        self.trace, self.compute = [], compute

    def fdb_kernel_create_mixed(self, desc, space2, out):
        d, s = me._obj(desc), me._obj(space2)
        if d.form not in _TRANSFERS:
            return self._fail("mock engine: only the p-multigrid transfers are emulated on two spaces")
        nf, nc = d.degree + 1, s.degree + 1
        P = np.array(s.B[:nf * nc]).reshape(nf, nc)
        R = np.array(d.B[:nc * nf]).reshape(nc, nf)
        self._next += 1
        self.kernels[self._next] = dict(kind=_TRANSFERS[d.form], p=d.degree, q=s.degree, cdim=d.cdim,
                                        P3=_kron3(P), R3=_kron3(R), offf=np.array(d.offset0[:nf ** 3]),
                                        offc=np.array(s.offset[:nc ** 3]))
        me._obj(out).value = self._next
        return 0

    def fdb_kernel_call(self, h, ca):
        k, a = self.kernels[me._addr(h)], me._obj(ca)
        if k["kind"] == "jit":
            self.trace.append(("jit", k["name"]))
        elif k["kind"] == "helmholtz":
            self.trace.append(("helmholtz", k["degree"], "diagonal" if k["diagonal"] else "action"))
        else:
            self.trace.append((k["kind"], k["p"], k["q"]))
            return self._call_transfer(k, a) if self.compute else 0
        return super().fdb_kernel_call(h, ca) if self.compute else 0

    def _call_transfer(self, k, a):
        """The kernels' semantics cell by cell: prolong and inject write, restrict adds P^T (w o fine)."""
        if a.location != _lib.LOC_DEVICE:
            return self._fail("p transfer: device mode only")
        nlay, ncols, cd = a.layers[1] - 1, a.end, k["cdim"]
        nf3, nc3 = len(k["offf"]), len(k["offc"])
        fm = 0 if k["kind"] == "p_prolong" else 1
        mapf = me._view(a.maps[fm], ncols * nf3, np.int32).reshape(ncols, nf3).astype(np.int64)
        mapc = me._view(a.maps[1 - fm], ncols * nc3, np.int32).reshape(ncols, nc3).astype(np.int64)
        lay = np.arange(nlay)
        ff = (mapf[:, None, :] + lay[None, :, None] * k["offf"]).reshape(-1, nf3)
        fc = (mapc[:, None, :] + lay[None, :, None] * k["offc"]).reshape(-1, nc3)
        nfine, ncoarse = int(ff.max()) + 1, int(fc.max()) + 1
        if k["kind"] == "p_prolong":
            fine = me._view(a.args[0], nfine * cd).reshape(nfine, cd)
            coarse = me._view(a.args[1], ncoarse * cd).reshape(ncoarse, cd)
            fine[ff] = np.einsum("ia,cak->cik", k["P3"], coarse[fc])
        elif k["kind"] == "p_inject":
            coarse = me._view(a.args[0], ncoarse * cd).reshape(ncoarse, cd)
            fine = me._view(a.args[1], nfine * cd).reshape(nfine, cd)
            coarse[fc] = np.einsum("ai,cik->cak", k["R3"], fine[ff])
        else:
            coarse = me._view(a.args[0], ncoarse * cd).reshape(ncoarse, cd)
            fine = me._view(a.args[1], nfine * cd).reshape(nfine, cd)
            w = me._view(a.args[2], nfine)
            np.add.at(coarse, fc, np.einsum("ia,cik->cak", k["P3"], w[ff][:, :, None] * fine[ff]))
        return 0

    def fdb_vec_chebyshev(self, n, cd, cz, b, ax, dinv, d, x):
        self.trace.append(("fdb_vec_chebyshev", int(n)))
        po.chebyshev_step(cd, cz, me._view(b, n), me._view(ax, n), me._view(dinv, n), me._view(d, n),
                          me._view(x, n))
        return 0


def _recorded(name):
    def f(self, *args):
        self.trace.append((name, int(args[0]) if name.startswith("fdb_vec") else None))
        return getattr(me.MockEngine, name)(self, *args)
    return f


for _n in _RECORDED:
    setattr(PMGEngine, _n, _recorded(_n))


class pmg_mock(me.install):
    def __init__(self, oracle, compute=True):
        self.engine = PMGEngine(oracle, compute)


def _problem(p, nx=3, ny=2, nz=3):
    V = FunctionSpace(ExtrudedHexMesh(nx, ny, nz, warp=0.05, permute_seed=2), p)
    return V, [DirichletBC(V, 0.0, s) for s in ("bottom", "top")]


@pytest.mark.parametrize("p", [2, 3])
@pytest.mark.parametrize("kind", ["firedrake.PMGPC", "firedrake.P1PC"])
def test_one_cycle_engine_calls(oracle, p, kind):
    """One cycle of a two-level PMG (CG_p over CG1), nu = 2 Chebyshev iterations: on the fine level one action and
    one fused pass per iteration, the residual, one restriction and one prolongation and nothing else; the coarse
    level is the Jacobi-PCG of its own space between them."""
    with pmg_mock(oracle) as eng:
        V, bcs = _problem(p)
        from firedrake_b200.assemble import _pmg
        pm = _pmg(V, lambda W, k=None: Form(W), {"pc_python_type": kind}, bcs, None, None)
        assert pm.degrees == [1, p]
        r = V.dat(np.sin(np.arange(V.node_count)))
        for bc in bcs:
            bc.zero(r)
        z = V.dat()
        pm.apply(pm.top, r, z)                  # first cycle: the transfer weights, the lazily zeroed work vectors
        z.zero()
        z.device_ptr
        eng.trace.clear()
        pm.apply(pm.top, r, z)
        trace = list(eng.trace)
        zmax = np.abs(z.data_ro).max()
    nf, nc = V.node_count, pm.spaces[0].node_count
    A, cheb = ("helmholtz", p, "action"), ("fdb_vec_chebyshev", nf)
    i_r, i_p = trace.index(("p_restrict", p, 1)), trace.index(("p_prolong", p, 1))
    assert [t[0] for t in trace].count("p_restrict") == 1 and [t[0] for t in trace].count("p_prolong") == 1
    assert not any(t[0] == "p_inject" for t in trace)
    zero_bc = [("fdb_dat_zero_nodes", None)] * len(bcs)
    # A.mult of the matrix-free operator with its Dirichlet rows: the one action among the vector operations
    mult = [("fdb_memcpy_d2d", None)] + zero_bc + [("fdb_memset", None), A] + [("fdb_dat_set_nodes", None)] * len(bcs)
    smooth = mult + [cheb] + mult + [cheb]
    assert trace[:i_r] == smooth + mult + [("fdb_vec_aypx", nf)] + zero_bc + [("fdb_memset", None)]
    # the coarse level: its right-hand side's boundary rows, x = 0, then Jacobi-PCG on CG1 alone
    coarse = trace[i_r + 1:i_p]
    assert coarse[:len(bcs)] == zero_bc
    assert all(t[1] in (nc, None) or t == ("helmholtz", 1, "action") for t in coarse), coarse
    assert ("helmholtz", 1, "action") in coarse and ("fdb_vec_pointwise_mult", nc) in coarse
    assert trace[i_p + 1:] == zero_bc + [("fdb_vec_axpy", nf)] + smooth
    assert zmax > 0.0


def test_mock_transfers_match_oracle(oracle):
    """The mock's transfers are the oracle's: prolong, restrict = P^T and inject on a permuted mesh."""
    with pmg_mock(oracle):
        mesh = ExtrudedHexMesh(3, 2, 2, warp=0.05, permute_seed=4)
        for p, q in ((2, 1), (3, 1), (3, 2)):
            Vc, Vf = FunctionSpace(mesh, q), FunctionSpace(mesh, p)
            T = mg.PTransfer(Vc, Vf)
            xc = np.random.default_rng(0).standard_normal(Vc.node_count)
            xf = np.random.default_rng(1).standard_normal(Vf.node_count)
            np.testing.assert_allclose(T.prolong(Vc.dat(xc), Vf.dat()).data_ro, po.prolong(Vf.V, Vc.V, xc),
                                       atol=1e-13)
            np.testing.assert_allclose(T.restrict(Vf.dat(xf), Vc.dat()).data_ro,
                                       po.restrict_cellwise(Vf.V, Vc.V, xf), atol=1e-13)
            np.testing.assert_allclose(T.inject(Vf.dat(xf), Vc.dat()).data_ro, po.inject(Vf.V, Vc.V, xf),
                                       atol=1e-13)


@pytest.mark.parametrize("p", [2, 3])
def test_iterations_on_mock(oracle, p):
    """The outer iterations of P1PC-CG on the mock engine, the same problem as tests/test_pmg_gpu.py::
    test_poisson_iterations (whose bounds are these counts): at most 2 more from 8^3 to 16^3, and at least 3x fewer
    than Jacobi-CG at 16^3."""
    its = {}
    for n in (8, 16):
        with pmg_mock(oracle):
            V = FunctionSpace(ExtrudedHexMesh(n, n, n, warp=0.05), p)
            bcs = [DirichletBC(V, 0.0, s) for s in ("bottom", "top")]
            L = assemble(mass(V), u=V.dat(np.sin(np.arange(V.node_count) * 0.37)))
            its[n], _ = solve(Form(V), L, V.dat(), bcs=bcs, solver_parameters=dict(P1, ksp_rtol=1e-11))
            if n == 16:
                its_j, _ = solve(Form(V), L, V.dat(), bcs=bcs, solver_parameters={"pc_type": "jacobi",
                                                                                   "ksp_rtol": 1e-11})
    assert its == {2: {8: 11, 16: 11}, 3: {8: 12, 16: 14}}[p]
    assert its[16] <= its[8] + 2 and 3 * its[16] <= its_j


def solve_engine_calls(oracle):
    """The engine calls of solve() with pc_type none, jacobi and mg on a small hierarchy, {pc_type: trace}, with the
    kernels recorded but not run: every vector stays zero, so the Krylov loops stop at once and the trace is the
    set-up and one application of the preconditioner (for mg one V-cycle), independent of rounding."""
    out = {}
    for pc in ("none", "jacobi", "mg"):
        with pmg_mock(oracle, compute=False) as eng:
            h = mg.MeshHierarchy(2, 2, 2, 1, warp=0.05)
            V = FunctionSpace(h[1], 2)
            bcs = [DirichletBC(V, 0.0, s) for s in ("bottom", "top")]
            L = assemble(mass(V), u=V.dat(np.cos(np.arange(V.node_count) * 0.3)))
            eng.trace.clear()
            solve(Form(V), L, V.dat(), bcs=bcs, hierarchy=h, solver_parameters={"pc_type": pc})
            out[pc] = [tuple(t) for t in eng.trace]
    return out


@pytest.mark.parametrize("pc", ["none", "jacobi", "mg"])
def test_gmg_paths_make_the_parent_calls(oracle, pc):
    """solve() with pc_type none, jacobi and mg makes the engine calls it made before p-multigrid: the V-cycle walk
    now shared with PMG (mg._LevelCycle.apply) included.  SOLVE_CALLS was recorded with solve_engine_calls() on the
    parent commit."""
    got = solve_engine_calls(oracle)[pc]
    assert got == [tuple(t) for t in SOLVE_CALLS[pc]]




# solve_engine_calls() run on the parent commit, the last one before p-multigrid: {pc_type: trace}
SOLVE_CALLS = \
{'jacobi': [('fdb_memset', None), ('fdb_dat_set_nodes_scalar', None), ('fdb_dat_set_nodes_scalar', None),
            ('fdb_memset', None), ('fdb_memcpy_d2d', None), ('fdb_dat_zero_nodes', None),
            ('fdb_dat_zero_nodes', None), ('fdb_memset', None), ('fdb_memset', None), ('helmholtz', 2, 'diagonal'),
            ('fdb_dat_set_nodes_scalar', None), ('fdb_dat_set_nodes_scalar', None), ('jit', 'recip'),
            ('fdb_memset', None), ('fdb_memcpy_d2d', None), ('fdb_dat_zero_nodes', None),
            ('fdb_dat_zero_nodes', None), ('fdb_memset', None), ('helmholtz', 2, 'action'),
            ('fdb_dat_set_nodes', None), ('fdb_dat_set_nodes', None), ('fdb_memset', None), ('fdb_memcpy_d2d', None),
            ('fdb_vec_axpy', 729), ('fdb_vec_dot', 729), ('fdb_memset', None), ('fdb_vec_pointwise_mult', 729),
            ('fdb_memset', None), ('fdb_memcpy_d2d', None), ('fdb_vec_dot', 729), ('fdb_dat_set_nodes_scalar', None),
            ('fdb_dat_set_nodes_scalar', None)],
 'mg': [('fdb_memset', None), ('fdb_dat_set_nodes_scalar', None), ('fdb_dat_set_nodes_scalar', None),
        ('fdb_memset', None), ('fdb_memcpy_d2d', None), ('fdb_dat_zero_nodes', None), ('fdb_dat_zero_nodes', None),
        ('fdb_memset', None), ('fdb_memset', None), ('helmholtz', 2, 'diagonal'), ('fdb_dat_set_nodes_scalar', None),
        ('fdb_dat_set_nodes_scalar', None), ('jit', 'recip'), ('fdb_memset', None), ('helmholtz', 2, 'diagonal'),
        ('fdb_dat_set_nodes_scalar', None), ('fdb_dat_set_nodes_scalar', None), ('jit', 'recip'),
        ('fdb_memset', None), ('fdb_memcpy_d2d', None), ('fdb_dat_zero_nodes', None), ('fdb_dat_zero_nodes', None),
        ('fdb_memset', None), ('helmholtz', 2, 'action'), ('fdb_dat_set_nodes', None), ('fdb_dat_set_nodes', None),
        ('fdb_memset', None), ('fdb_memcpy_d2d', None), ('fdb_vec_axpy', 729), ('fdb_vec_dot', 729),
        ('fdb_memset', None), ('fdb_memset', None), ('fdb_memcpy_d2d', None), ('fdb_dat_zero_nodes', None),
        ('fdb_dat_zero_nodes', None), ('fdb_memset', None), ('helmholtz', 2, 'action'), ('fdb_dat_set_nodes', None),
        ('fdb_dat_set_nodes', None), ('fdb_vec_aypx', 729), ('fdb_vec_pointwise_mult', 729), ('fdb_vec_axpy', 729),
        ('fdb_memcpy_d2d', None), ('fdb_dat_zero_nodes', None), ('fdb_dat_zero_nodes', None), ('fdb_memset', None),
        ('helmholtz', 2, 'action'), ('fdb_dat_set_nodes', None), ('fdb_dat_set_nodes', None), ('fdb_vec_aypx', 729),
        ('fdb_vec_pointwise_mult', 729), ('fdb_vec_axpy', 729), ('fdb_memcpy_d2d', None),
        ('fdb_dat_zero_nodes', None), ('fdb_dat_zero_nodes', None), ('fdb_memset', None), ('helmholtz', 2, 'action'),
        ('fdb_dat_set_nodes', None), ('fdb_dat_set_nodes', None), ('fdb_vec_aypx', 729), ('fdb_dat_zero_nodes', None),
        ('fdb_dat_zero_nodes', None), ('fdb_memset', None), ('fdb_memset', None), ('jit', 'count'), ('jit', 'recip'),
        ('jit', 'restrict_'), ('fdb_dat_zero_nodes', None), ('fdb_dat_zero_nodes', None), ('fdb_memset', None),
        ('fdb_memset', None), ('fdb_memcpy_d2d', None), ('fdb_dat_zero_nodes', None), ('fdb_dat_zero_nodes', None),
        ('fdb_memset', None), ('helmholtz', 2, 'action'), ('fdb_dat_set_nodes', None), ('fdb_dat_set_nodes', None),
        ('fdb_memset', None), ('fdb_memcpy_d2d', None), ('fdb_vec_axpy', 125), ('fdb_memset', None),
        ('fdb_memcpy_d2d', None), ('fdb_vec_dot', 125), ('fdb_memset', None), ('jit', 'prolong'),
        ('fdb_dat_zero_nodes', None), ('fdb_dat_zero_nodes', None), ('fdb_vec_axpy', 729), ('fdb_memcpy_d2d', None),
        ('fdb_dat_zero_nodes', None), ('fdb_dat_zero_nodes', None), ('fdb_memset', None), ('helmholtz', 2, 'action'),
        ('fdb_dat_set_nodes', None), ('fdb_dat_set_nodes', None), ('fdb_vec_aypx', 729),
        ('fdb_vec_pointwise_mult', 729), ('fdb_vec_axpy', 729), ('fdb_memcpy_d2d', None),
        ('fdb_dat_zero_nodes', None), ('fdb_dat_zero_nodes', None), ('fdb_memset', None), ('helmholtz', 2, 'action'),
        ('fdb_dat_set_nodes', None), ('fdb_dat_set_nodes', None), ('fdb_vec_aypx', 729),
        ('fdb_vec_pointwise_mult', 729), ('fdb_vec_axpy', 729), ('fdb_memset', None), ('fdb_memcpy_d2d', None),
        ('fdb_vec_dot', 729), ('fdb_dat_set_nodes_scalar', None), ('fdb_dat_set_nodes_scalar', None)],
 'none': [('fdb_memset', None), ('fdb_dat_set_nodes_scalar', None), ('fdb_dat_set_nodes_scalar', None),
          ('fdb_memset', None), ('fdb_memcpy_d2d', None), ('fdb_dat_zero_nodes', None), ('fdb_dat_zero_nodes', None),
          ('fdb_memset', None), ('fdb_memset', None), ('fdb_memcpy_d2d', None), ('fdb_dat_zero_nodes', None),
          ('fdb_dat_zero_nodes', None), ('fdb_memset', None), ('helmholtz', 2, 'action'), ('fdb_dat_set_nodes', None),
          ('fdb_dat_set_nodes', None), ('fdb_memset', None), ('fdb_memcpy_d2d', None), ('fdb_vec_axpy', 729),
          ('fdb_memset', None), ('fdb_memcpy_d2d', None), ('fdb_vec_dot', 729), ('fdb_dat_set_nodes_scalar', None),
          ('fdb_dat_set_nodes_scalar', None)]}
