"""Geometric multigrid on extruded hex hierarchies (SURVEY.md section 8f row f3):
``prolong`` / ``restrict`` / ``inject`` and a matrix-free V-cycle.

Reference: firedrake/mg/interface.py:37-113 (prolong), :116-190 (restrict),
:193-280 (inject), kernels firedrake/mg/kernels.py:157-380.  The reference loops
over FINE NODES; each one locates itself in a coarse cell by a Newton iteration
on the coarse coordinate field and evaluates the coarse basis there.  For the
nested hierarchies produced by uniform refinement that search always lands on
the parent cell at a reference position known a priori, so here the loops run
over COARSE CELLS and apply 1-D transfer matrices by sum factorisation:

    prolong   fine[(2p+1)^3 lattice of the 8 children] = (P (x) P (x) P) coarse      WRITE
    restrict  coarse += (P (x) P (x) P)^T (fine / multiplicity)                      INC
    inject    coarse[a] = fine function evaluated at coarse node a                   WRITE

``P[i][a]`` = coarse 1-D basis function a at fine lattice position i.  The transfer
kernels are generated C run through the engine's generic wrapper builder
(codegen.py / csrc/wrapper_jit.cu), with a coarse-cell -> fine-node map whose
layer offset is twice the fine space's (one coarse layer = two fine layers).

Status: kernels and maps are CPU-verified (tests/test_mg.py: polynomial
exactness, restrict == prolong^T, inject o prolong == id); the V-cycle logic is
CPU-verified against a mock engine (tests/test_host_logic_mock.py: level-independent
contraction ~0.12 for CG1, ~0.19 for CG2, PCG in 6-8 iterations on 4^3..32^3) and runs on
the GPU (tests/test_jit_gpu.py::test_mg_*, benchmarks/mg_solve.py).
"""
from __future__ import annotations

import numpy as np

from . import op2
from .codegen import CStringKernel
from .fiat_lite import _lagrange_tab, interval_element


# ------------------------------------------------------------------ 1-D tables
def fine_lattice_positions(p):
    """Positions on the COARSE reference interval of the 2p+1 fine nodes of its two
    children, ascending (child c holds GLL node m at (c + gll[m]) / 2)."""
    gll = np.sort(interval_element(p).nodes)
    return np.concatenate([gll / 2.0, (1.0 + gll[1:]) / 2.0])


def prolongation_matrix(p):
    """(2p+1, p+1): coarse basis a (dof numbering) at fine lattice position i."""
    B, _ = _lagrange_tab(interval_element(p).nodes, fine_lattice_positions(p))
    return B


def injection_matrix(p):
    """(p+1, 2p+1): value at coarse node a (dof numbering) of the fine piecewise
    polynomial with lattice coefficients; a node on the children's interface is
    evaluated in child 0."""
    el = interval_element(p)
    gll = np.sort(el.nodes)
    J = np.zeros((p + 1, 2 * p + 1))
    for a, xc in enumerate(el.nodes):
        c = 0 if xc <= 0.5 else 1
        xi = 2.0 * xc - c                                  # position inside child c
        B, _ = _lagrange_tab(gll, np.array([xi]))          # child basis, ascending positions
        J[a, c * p:c * p + p + 1] = B[0]
    J[np.abs(J) < 1e-15] = 0.0
    return J


def _table(a):
    a = np.asarray(a)
    if a.ndim == 1:
        return "{" + ", ".join(repr(float(v)) for v in a) + "}"
    return "{" + ", ".join(_table(r) for r in a) + "}"


_TENSOR = """
/* out[(i*NO+j)*NO+k][c] = sum_{a,b,d} T[i][a] T[j][b] T[k][d] in[(a*NI+b)*NI+d][c], by sum factorisation */
static inline void %(name)s_apply(const double T[%(NO)d][%(NI)d], const double *in, double *out)
{
    double t1[%(NO)d * %(NI)d * %(NI)d * %(CD)d], t2[%(NO)d * %(NO)d * %(NI)d * %(CD)d];
    for (int i = 0; i < %(NO)d; ++i)
        for (int r = 0; r < %(NI)d * %(NI)d * %(CD)d; ++r) {
            double s = 0.0;
            for (int a = 0; a < %(NI)d; ++a) s += T[i][a] * in[a * %(NI)d * %(NI)d * %(CD)d + r];
            t1[i * %(NI)d * %(NI)d * %(CD)d + r] = s;
        }
    for (int i = 0; i < %(NO)d; ++i)
        for (int j = 0; j < %(NO)d; ++j)
            for (int r = 0; r < %(NI)d * %(CD)d; ++r) {
                double s = 0.0;
                for (int b = 0; b < %(NI)d; ++b) s += T[j][b] * t1[(i * %(NI)d + b) * %(NI)d * %(CD)d + r];
                t2[(i * %(NO)d + j) * %(NI)d * %(CD)d + r] = s;
            }
    for (int ij = 0; ij < %(NO)d * %(NO)d; ++ij)
        for (int k = 0; k < %(NO)d; ++k)
            for (int c = 0; c < %(CD)d; ++c) {
                double s = 0.0;
                for (int d = 0; d < %(NI)d; ++d) s += T[k][d] * t2[(ij * %(NI)d + d) * %(CD)d + c];
                out[(ij * %(NO)d + k) * %(CD)d + c] = s;
            }
}
"""


def prolong_kernel(p, cdim=1):
    n, m = p + 1, 2 * p + 1
    code = (f"static const double PRO[{m}][{n}] = {_table(prolongation_matrix(p))};\n"
            + _TENSOR % dict(name="prolong", NO=m, NI=n, CD=cdim)
            + f"""
static void prolong(double *fine, const double *coarse)
{{
    prolong_apply(PRO, coarse, fine);
}}
""")
    return CStringKernel(code, "prolong")


def restrict_kernel(p, cdim=1):
    """coarse (INC) += P^T (fine * weight): ``weight`` = 1 / (number of coarse cells whose
    lattice contains the fine node), so that every fine node contributes exactly once --
    the reference attributes each fine node to one coarse cell instead
    (firedrake/mg/utils.py fine_node_to_coarse_node_map)."""
    n, m = p + 1, 2 * p + 1
    code = (f"static const double PROT[{n}][{m}] = {_table(prolongation_matrix(p).T)};\n"
            + _TENSOR % dict(name="restrict", NO=n, NI=m, CD=cdim)
            + f"""
static void restrict_(double *coarse, const double *fine, const double *weight)
{{
    double w[{m ** 3 * cdim}], r[{n ** 3 * cdim}];
    for (int i = 0; i < {m ** 3}; ++i)
        for (int c = 0; c < {cdim}; ++c) w[i * {cdim} + c] = fine[i * {cdim} + c] * weight[i];
    restrict_apply(PROT, w, r);
    for (int i = 0; i < {n ** 3 * cdim}; ++i) coarse[i] += r[i];
}}
""")
    return CStringKernel(code, "restrict_")


def inject_kernel(p, cdim=1):
    n, m = p + 1, 2 * p + 1
    code = (f"static const double INJ[{n}][{m}] = {_table(injection_matrix(p))};\n"
            + _TENSOR % dict(name="inject", NO=n, NI=m, CD=cdim)
            + f"""
static void inject(double *coarse, const double *fine)
{{
    inject_apply(INJ, fine, coarse);
}}
""")
    return CStringKernel(code, "inject")


# ------------------------------------------------------------------- hierarchy
def coarse_to_fine_node_map(Vc, Vf):
    """(coarse columns, (2p+1)^3) fine node of every lattice point of the BOTTOM coarse
    cell of each column, lattice order (i*(2p+1)+j)*(2p+1)+k, and the per-coarse-layer
    offsets.  ``Vc``/``Vf``: ExtrudedFunctionSpaces of the same degree on a mesh and
    its uniform refinement (2x in x, y and layers)."""
    mc, mf = Vc.mesh, Vf.mesh
    p, n = Vc.degree, Vc.degree + 1
    if (mf.nx, mf.ny, mf.nz) != (2 * mc.nx, 2 * mc.ny, 2 * mc.nz) or Vf.degree != p:
        raise ValueError("Vf must be the same space on the uniform refinement of Vc's mesh")
    fcol = np.full((mf.nx, mf.ny), -1, dtype=np.int64)
    fcol[mf.cell_ix, mf.cell_iy] = np.arange(mf.num_base_cells)
    pos2dof = np.empty(n, dtype=np.int64)
    pos2dof[np.array([0, n - 1] + list(range(1, n - 1)))] = np.arange(n)    # ascending position -> dof
    m = 2 * p + 1
    child = np.where(np.arange(m) <= p, 0, 1)                # lattice index -> child, local position
    lpos = np.arange(m) - child * p
    ldof = pos2dof[lpos]
    values = np.empty((mc.num_base_cells, m ** 3), dtype=np.int32)
    offset = np.empty(m ** 3, dtype=np.int32)
    fmap, foff = Vf.cell_node_map.astype(np.int64), np.asarray(Vf.offset, dtype=np.int64)
    for i in range(m):
        for j in range(m):
            cols = fcol[2 * mc.cell_ix + child[i], 2 * mc.cell_iy + child[j]]
            for k in range(m):
                loc = (ldof[i] * n + ldof[j]) * n + ldof[k]
                L = (i * m + j) * m + k
                values[:, L] = fmap[cols, loc] + foff[loc] * child[k]
                offset[L] = 2 * foff[loc]
    return values, offset


class TransferManager:
    """prolong / restrict / inject between two consecutive levels
    (firedrake/mg/embedded.py TransferManager, firedrake/mg/interface.py)."""

    def __init__(self, Vc, Vf):
        """``Vc``, ``Vf``: assemble.FunctionSpace on consecutive levels."""
        self.Vc, self.Vf = Vc, Vf
        p = Vc.degree
        vals, off = coarse_to_fine_node_map(Vc.V, Vf.V)
        self.c2f = op2.Map(Vc.cell_set, Vf.node_set, (2 * p + 1) ** 3, vals, offset=off, name="coarse_to_fine")
        self._k = (prolong_kernel(p, Vc.cdim), restrict_kernel(p, Vc.cdim), inject_kernel(p, Vc.cdim))
        self._weight = None

    @property
    def weight(self):
        """1 / multiplicity of every fine node in the coarse-cell lattices (scalar Dat)."""
        if self._weight is None:
            # scalar field on the fine nodes, sharing the fine space's halo: the counts of nodes on
            # a slab interface are summed into their owner and sent back to the ghost copies
            w = op2.Dat(op2.DataSet(self.Vf.node_set, 1, halo=self.Vf.dof_dset.halo))
            m3 = (2 * self.Vc.degree + 1) ** 3
            count = CStringKernel(f"static void count(double *w) {{ for (int i = 0; i < {m3}; ++i) w[i] += 1.0; }}",
                                  "count")
            op2.par_loop(count, self.Vc.cell_set, w(op2.INC, self.c2f))
            inv = CStringKernel("static void recip(double *w) { *w = 1.0 / *w; }", "recip")
            op2.par_loop(inv, self.Vf.node_set, w(op2.RW))
            self._weight = w
        return self._weight

    def prolong(self, coarse: op2.Dat, fine: op2.Dat):
        op2.par_loop(self._k[0], self.Vc.cell_set, fine(op2.WRITE, self.c2f),
                     coarse(op2.READ, self.Vc.cell_node_map))
        return fine

    def restrict(self, fine_dual: op2.Dat, coarse_dual: op2.Dat):
        coarse_dual.zero()
        coarse_dual.device_ptr                      # materialise the zero on the device
        op2.par_loop(self._k[1], self.Vc.cell_set, coarse_dual(op2.INC, self.Vc.cell_node_map),
                     fine_dual(op2.READ, self.c2f), self.weight(op2.READ, self.c2f))
        return coarse_dual

    def inject(self, fine: op2.Dat, coarse: op2.Dat):
        op2.par_loop(self._k[2], self.Vc.cell_set, coarse(op2.WRITE, self.Vc.cell_node_map),
                     fine(op2.READ, self.c2f))
        return coarse


def prolong(coarse, fine, manager):
    return manager.prolong(coarse, fine)


def restrict(fine_dual, coarse_dual, manager):
    return manager.restrict(fine_dual, coarse_dual)


def inject(fine, coarse, manager):
    return manager.inject(fine, coarse)


def reciprocal_kernel(cdim=1):
    """Node kernel inverting every one of the ``cdim`` components of a RW Dat in place (the Jacobi
    preconditioner's inverse diagonal)."""
    if cdim == 1:
        return CStringKernel("static void recip(double *w) { *w = 1.0 / *w; }", "recip")
    return CStringKernel(f"static void recip{cdim}(double *w) {{ for (int c = 0; c < {cdim}; ++c) w[c] = 1.0 / w[c]; }}",
                         f"recip{cdim}")


def _touched(*dats):
    """Vector algebra ran over the local entries: owned rows are right, ghost rows are not
    (pyop2/types/dat.py:622-678: any write invalidates the halo)."""
    for d in dats:
        d._device_written()
        d.halo_valid = False


# --------------------------------------------------------------------- V-cycle
class MeshHierarchy:
    """``ExtrudedMeshHierarchy`` of uniformly refined extruded hex meshes
    (firedrake/mg/mesh.py:190-260): level l has 2^l times the coarse resolution in
    every direction."""

    def __init__(self, nx, ny, nz, levels, rank=0, nranks=1, **mesh_kwargs):
        """``rank`` / ``nranks``: this process's slab of every level (firedrake_b200.partition); the
        coarse slab bounds must refine exactly (``nx`` divisible by ``nranks``) so that every
        coarse cell's children live on the same rank, as in a refined DMPlex distribution."""
        from .utility_meshes import ExtrudedHexMesh
        self.partitions = None
        if nranks > 1:
            if nx % nranks:
                raise ValueError("coarse nx must be divisible by the number of ranks")
            self.nranks, self.rank = nranks, rank
            self._sizes = [(nx << l, ny << l, nz << l) for l in range(levels + 1)]
            self._kwargs = mesh_kwargs
            self.partitions = {}
            self.meshes = [None] * (levels + 1)
            return
        self.meshes = [ExtrudedHexMesh(nx << l, ny << l, nz << l, **mesh_kwargs) for l in range(levels + 1)]

    def partition(self, level, degree):
        """SlabPartition of ``level`` for function spaces of ``degree`` (built on demand)."""
        from .partition import SlabPartition
        key = (level, degree)
        if key not in self.partitions:
            nx, ny, nz = self._sizes[level]
            self.partitions[key] = SlabPartition(nx, ny, nz, degree, self.rank, self.nranks, **self._kwargs)
            self.meshes[level] = self.partitions[key].mesh
        return self.partitions[key]

    def __len__(self):
        return len(self.meshes)

    def __getitem__(self, i):
        return self.meshes[i]


class _LevelCycle:
    """The multigrid cycle shared by :class:`VCycle` (levels = meshes) and :class:`PMG` (levels = degrees on one
    mesh): pre-smooth, residual, restrict, coarse correction, prolong, post-smooth, one level at a time.  A subclass
    sets ``ops``, ``bcs``, ``transfers``, ``invdiag``, ``_work`` (per level: r, e, t, b, x) and ``nu`` / ``omega``, and
    provides ``_coarse_solve``; ``_smooth`` defaults to damped Jacobi."""

    def _smooth(self, l, b, x):
        """x += omega D^-1 (b - A x), nu times."""
        from . import _lib
        L = _lib.lib()
        A, w = self.ops[l], self._work[l]
        n = b._data.size
        for _ in range(self.nu):
            A.mult(x, w["t"])
            _lib.check(L.fdb_vec_aypx(n, -1.0, b.device_ptr, w["t"].device_ptr))        # t = b - A x
            _lib.check(L.fdb_vec_pointwise_mult(n, w["t"].device_ptr, self.invdiag[l].device_ptr,
                                                w["t"].device_ptr))
            _touched(w["t"])
            _lib.check(L.fdb_vec_axpy(n, self.omega, w["t"].device_ptr, x.device_ptr))
            _touched(x)

    def apply(self, l, b, x):
        """One cycle on level l for A x = b, starting from the x passed in."""
        from . import _lib
        L = _lib.lib()
        A, w = self.ops[l], self._work[l]
        n = b._data.size
        if l == 0:
            self._coarse_solve(b, x)
            return x
        self._smooth(l, b, x)
        A.mult(x, w["r"])
        _lib.check(L.fdb_vec_aypx(n, -1.0, b.device_ptr, w["r"].device_ptr))             # r = b - A x
        _touched(w["r"])
        for bc in self.bcs[l]:
            bc.zero(w["r"])
        wc = self._work[l - 1]
        T = self.transfers[l - 1]
        T.restrict(w["r"], wc["b"])
        for bc in self.bcs[l - 1]:
            bc.zero(wc["b"])
        wc["x"].zero()
        wc["x"].device_ptr
        self.apply(l - 1, wc["b"], wc["x"])
        T.prolong(wc["x"], w["e"])
        for bc in self.bcs[l]:
            bc.zero(w["e"])
        _lib.check(L.fdb_vec_axpy(n, 1.0, w["e"].device_ptr, x.device_ptr))
        _touched(x)
        self._smooth(l, b, x)
        return x


class VCycle(_LevelCycle):
    """Matrix-free geometric multigrid V-cycle for the Helmholtz family with rediscretised
    coarse operators (the ``pc_type mg`` + ``mat_type matfree`` setup of
    demos/multigrid/geometric_multigrid.py.rst): damped-Jacobi smoothing with the
    assembled diagonal (``ImplicitMatrixContext.getDiagonal``, operators.py:199-205),
    coarsest level solved by CG.  Everything stays on the device."""

    def __init__(self, hierarchy, degree, make_form, bc_domains=(), nu=2, omega=0.8,
                 coarse_rtol=1e-2, coarse_maxit=200, allreduce=None, kappa=None, cdim=1):
        """``allreduce``: callable summing a float over the ranks (partitioned hierarchies).
        ``kappa``: coefficient field on the finest level (a scalar Dat laid out like this V-cycle's
        finest space); it is copied there, each coarser level gets the injection of the next finer
        level's field, and the operators are ``make_form(V, kappa_l)``.  ``cdim``: value size of the
        level spaces (3 for elasticity); Dirichlet conditions constrain every component."""
        from .assemble import DirichletBC, FunctionSpace, assemble
        self.allreduce = allreduce
        if hierarchy.partitions is None:
            self.spaces = [FunctionSpace(m, degree, cdim) for m in hierarchy.meshes]
        else:
            parts = [hierarchy.partition(l, degree) for l in range(len(hierarchy))]
            self.spaces = [FunctionSpace(pt.mesh, degree, cdim, partition=pt) for pt in parts]
        self.bcs = [[DirichletBC(V, 0.0, s) for s in bc_domains] for V in self.spaces]
        self.transfers = [TransferManager(self.spaces[l], self.spaces[l + 1]) for l in range(len(self.spaces) - 1)]
        if kappa is None:
            forms = [make_form(V) for V in self.spaces]
        else:
            self.kappas = self._coarsen_coefficient(kappa)
            forms = [make_form(V, k) for V, k in zip(self.spaces, self.kappas)]
        for f in forms:
            if getattr(f.V, "family", "CG") == "DQ":
                raise NotImplementedError("VCycle does not take DQ spaces: its transfers and smoothers are those of "
                                          "nested CG spaces; DQ solves take pc_type 'none' or 'jacobi'")
        self.ops = [assemble(f, bcs=b, mat_type="matfree") for f, b in zip(forms, self.bcs)]
        self.nu, self.omega = nu, omega
        self.coarse_rtol, self.coarse_maxit = coarse_rtol, coarse_maxit
        self.invdiag = []
        for V, A in zip(self.spaces, self.ops):
            d = A.getDiagonal(V.dat())
            op2.par_loop(reciprocal_kernel(cdim), V.node_set, d(op2.RW))
            self.invdiag.append(d)
        # per level: r residual, t smoother scratch, e prolonged correction; as a COARSE level also
        # b (restricted residual = its right-hand side) and x (its solution) -- x and e must be
        # distinct Dats: level l-1's solution is the input of the prolongation into level l's e
        self._work = [dict(r=V.dat(), e=V.dat(), t=V.dat(), b=V.dat(), x=V.dat()) for V in self.spaces]

    def _coarsen_coefficient(self, kappa):
        """kappa on every level, finest last: the finest is a device copy of ``kappa`` on this
        V-cycle's own space, each coarser one the injection of the next finer."""
        from . import _lib
        top = self.spaces[-1]
        fine = top.dat()
        if kappa.nbytes != fine.nbytes:
            raise ValueError("kappa does not match the finest level of the hierarchy")
        _lib.check(_lib.lib().fdb_memcpy_d2d(fine.device_ptr, kappa.device_ptr, kappa.nbytes))
        _touched(fine)
        out = [fine]
        for l in range(len(self.spaces) - 2, -1, -1):
            out.insert(0, self.transfers[l].inject(out[0], self.spaces[l].dat()))
        return out

    def _coarse_solve(self, b, x):
        """The coarsest level: CG to ``coarse_rtol``."""
        from .assemble import cg
        cg(self.ops[0], b, x, rtol=self.coarse_rtol, maxit=self.coarse_maxit, allreduce=self.allreduce)
        _touched(x)


def pcg(A, b, x, M, rtol=1e-8, maxit=200, allreduce=None):
    """Preconditioned CG (``ksp_type cg`` with a multigrid ``pc``): ``M(r, z)`` applies the
    preconditioner (e.g. ``lambda r, z: vcycle.apply(top, r, z)`` from z = 0).  ``allreduce``:
    callable summing a float over the ranks; inner products then run over the OWNED dofs."""
    import ctypes as C
    from . import _lib
    L = _lib.lib()
    V = b.dataset
    r, z, p, Ap = (op2.Dat(V) for _ in range(4))
    n = b._data.size
    n_owned = b.dataset.set.size * b.cdim

    def dot(u, v):
        out = C.c_double()
        _lib.check(L.fdb_vec_dot(n_owned, u.device_ptr, v.device_ptr, C.byref(out)))
        return allreduce(out.value) if allreduce else out.value
    A.mult(x, Ap)
    _lib.check(L.fdb_memcpy_d2d(r.device_ptr, b.device_ptr, b.nbytes))
    r._device_written()
    _lib.check(L.fdb_vec_axpy(n, -1.0, Ap.device_ptr, r.device_ptr))
    _touched(r)
    r0 = np.sqrt(dot(r, r))
    hist = [r0]
    z.zero(); z.device_ptr
    M(r, z)
    _lib.check(L.fdb_memcpy_d2d(p.device_ptr, z.device_ptr, z.nbytes))
    p._device_written()
    rz = dot(r, z)
    it = 0
    while it < maxit and hist[-1] > rtol * r0:
        A.mult(p, Ap)
        alpha = rz / dot(p, Ap)
        _lib.check(L.fdb_vec_axpy(n, alpha, p.device_ptr, x.device_ptr))
        _lib.check(L.fdb_vec_axpy(n, -alpha, Ap.device_ptr, r.device_ptr))
        _touched(x, r)
        hist.append(np.sqrt(dot(r, r)))
        z.zero(); z.device_ptr
        M(r, z)
        rz_new = dot(r, z)
        _lib.check(L.fdb_vec_aypx(n, rz_new / rz, z.device_ptr, p.device_ptr))            # p = z + beta p
        _touched(p)
        rz = rz_new
        it += 1
    return it, hist


# ------------------------------------------------------------------ p-multigrid
class PTransfer:
    """prolong / restrict / inject between two degrees on ONE mesh, CG_q (``Vc``) and CG_p (``Vf``), q < p, with
    :class:`TransferManager`'s interface, on the hand-written kernels of csrc/p_transfer_hex.cu (forms "p_prolong",
    "p_restrict", "p_inject").  The pairs (p, q) are (2, 1), (3, 1) and (3, 2); the engine refuses the others.
    ``scatter``: "atomic" or "coloured" (bit-reproducible) for the restriction."""

    def __init__(self, Vc, Vf, scatter="atomic"):
        for W in (Vc, Vf):
            if getattr(W, "family", "CG") == "NCF":
                raise NotImplementedError("PTransfer does not take NCF (H(div)) spaces: the only form on NCF is "
                                          "MixedPoisson")
            if getattr(W, "family", "CG") != "CG":
                raise NotImplementedError("PTransfer: CG spaces only (there is no DQ p-multigrid)")
        if Vc.mesh is not Vf.mesh or Vc.cdim != Vf.cdim or not Vc.degree < Vf.degree:
            raise ValueError("PTransfer: Vc and Vf must be spaces of one value size on the same mesh, Vc of the "
                             "lower degree")
        if Vf.dof_dset.halo is not None or Vc.dof_dset.halo is not None:
            raise NotImplementedError("PTransfer: partitioned spaces are not supported")
        self.Vc, self.Vf, self.scatter = Vc, Vf, scatter
        # the coarse rows on the fine space's cell set: every loop iterates Vf.cell_set
        self.cmap = op2.Map(Vf.cell_set, Vc.node_set, Vc.V.arity, Vc.V.cell_node_map, offset=Vc.V.offset,
                            name="p_coarse")
        kw = dict(degree=Vf.degree, coarse_degree=Vc.degree, cdim=Vf.cdim)
        self._k = {f: op2.Kernel(f, **kw) for f in ("p_prolong", "p_restrict", "p_inject")}
        self._gk = {}
        self._weight = None

    @property
    def weight(self):
        """1 / (number of cells containing the fine node), a scalar Dat on the fine nodes: set-up only, so it runs
        on the generic wrapper path."""
        if self._weight is None:
            w = op2.Dat(op2.DataSet(self.Vf.node_set, 1))
            nd = self.Vf.V.arity
            count = CStringKernel(f"static void count(double *w) {{ for (int i = 0; i < {nd}; ++i) w[i] += 1.0; }}",
                                  "count")
            op2.par_loop(count, self.Vf.cell_set, w(op2.INC, self.Vf.cell_node_map))
            op2.par_loop(reciprocal_kernel(1), self.Vf.node_set, w(op2.RW))
            self._weight = w
        return self._weight

    def _loop(self, form, *args):
        gk = self._gk.get(form)
        if gk is None:
            maps = []
            for a in args:
                if a.map not in maps:
                    maps.append(a.map)
            gk = self._gk[form] = op2.GlobalKernel(self._k[form], maps, extruded=True,
                                                   scatter=self.scatter if form == "p_restrict" else "atomic")
        op2.Parloop(gk, self.Vf.cell_set, args)()

    def prolong(self, coarse: op2.Dat, fine: op2.Dat):
        self._loop("p_prolong", fine(op2.WRITE, self.Vf.cell_node_map), coarse(op2.READ, self.cmap))
        return fine

    def restrict(self, fine_dual: op2.Dat, coarse_dual: op2.Dat):
        w = self.weight
        coarse_dual.zero()
        coarse_dual.device_ptr                      # materialise the zero on the device
        self._loop("p_restrict", coarse_dual(op2.INC, self.cmap), fine_dual(op2.READ, self.Vf.cell_node_map),
                   w(op2.READ, self.Vf.cell_node_map))
        return coarse_dual

    def inject(self, fine: op2.Dat, coarse: op2.Dat):
        self._loop("p_inject", coarse(op2.WRITE, self.cmap), fine(op2.READ, self.Vf.cell_node_map))
        return coarse


def pmg_degrees(p, coarse_degree=1, halve=True):
    """The level degrees of p-multigrid, coarsest first: PMGPC halves the degree (p -> max(p // 2, coarse)), P1PC
    (``halve=False``) goes straight to the coarse degree."""
    degs = [p]
    while degs[-1] > coarse_degree:
        degs.append(max(degs[-1] // 2, coarse_degree) if halve else coarse_degree)
    return degs[::-1]


def jacobi_lanczos_bounds(A, invdiag, b, steps=10, M=None):
    """The extreme eigenvalues (lmin, lmax) of D^-1 A estimated by ``steps`` Jacobi-preconditioned CG steps from the right-hand
    side ``b`` (PETSc's KSPChebyshev estimate): the CG coefficients give the Lanczos tridiagonal, whose extreme
    eigenvalues are computed on the host.  ``M(r, z)``: another preconditioner, writing z = P^-1 r (``invdiag`` is
    then not used); the estimate is then of P^-1 A."""
    import ctypes as C
    from . import _lib
    if steps < 1:
        raise ValueError(f"jacobi_lanczos_bounds: steps must be at least 1, got {steps}")
    L = _lib.lib()
    V = b.dataset
    r, z, p, Ap = (op2.Dat(V) for _ in range(4))
    n = b._data.size

    def dot(u, v):
        out = C.c_double()
        _lib.check(L.fdb_vec_dot(n, u.device_ptr, v.device_ptr, C.byref(out)))
        return out.value
    if M is None:
        def M(r, z):
            _lib.check(L.fdb_vec_pointwise_mult(n, r.device_ptr, invdiag.device_ptr, z.device_ptr))
    _lib.check(L.fdb_memcpy_d2d(r.device_ptr, b.device_ptr, b.nbytes))
    _touched(r)
    M(r, z)
    _touched(z)
    _lib.check(L.fdb_memcpy_d2d(p.device_ptr, z.device_ptr, z.nbytes))
    _touched(p)
    rz = dot(r, z)
    alphas, betas = [], []
    for _ in range(steps):
        A.mult(p, Ap)
        pAp = dot(p, Ap)
        if not pAp > 0.0:
            break
        alpha = rz / pAp
        _lib.check(L.fdb_vec_axpy(n, -alpha, Ap.device_ptr, r.device_ptr))
        M(r, z)
        _touched(r, z)
        rz_new = dot(r, z)
        alphas.append(alpha)
        betas.append(rz_new / rz)
        if not rz_new > 0.0:
            break
        _lib.check(L.fdb_vec_aypx(n, rz_new / rz, z.device_ptr, p.device_ptr))           # p = z + beta p
        _touched(p)
        rz = rz_new
    k = len(alphas)
    if k == 0:
        raise ArithmeticError(f"Chebyshev eigenvalue estimate: p.A p = {pAp} at the first step (P^-1 A is not "
                              f"positive definite, or the right-hand side is zero)")
    T = np.zeros((k, k))
    for j in range(k):
        T[j, j] = 1.0 / alphas[j] + (betas[j - 1] / alphas[j - 1] if j else 0.0)
        if j + 1 < k:
            T[j, j + 1] = T[j + 1, j] = np.sqrt(betas[j]) / alphas[j]
    ev = np.linalg.eigvalsh(T)
    return float(ev[0]), float(ev[-1])


def chebyshev_coefficients(emin, emax, k):
    """(c_d, c_z) of the k iterations d = c_d d + c_z D^-1 (b - A x), x += d of the Chebyshev iteration for D^-1 A
    with spectrum bounds [emin, emax] (Saad, Iterative Methods for Sparse Linear Systems, Algorithm 12.1); the first
    has c_d = 0."""
    theta, delta = 0.5 * (emax + emin), 0.5 * (emax - emin)
    sigma = theta / delta
    rho = 1.0 / sigma
    out = [(0.0, 1.0 / theta)]
    for _ in range(k - 1):
        rho_new = 1.0 / (2.0 * sigma - rho)
        out.append((rho_new * rho, 2.0 * rho_new / delta))
        rho = rho_new
    return out


class _SmoothedCycle(_LevelCycle):
    """The parts of a cycle with Chebyshev- or Richardson-Jacobi smoothing and a CG / V-cycle coarse solve, shared by
    :class:`PMG` and :class:`GTMG`.  A subclass sets, besides :class:`_LevelCycle`'s attributes, ``smoother``,
    ``stars`` (None per level, or a vertex-star relaxation), ``bounds`` (:meth:`_estimate_bounds`), ``coarse_mg`` /
    ``_coarse_top``, ``coarse_pc``, ``coarse_rtol``, ``coarse_maxit`` and a work vector "d" on every level."""

    def _estimate_bounds(self, esteig, esteig_steps, seed):
        """The Chebyshev bounds [a lmin + b lmax, c lmin + d lmax] of P^-1 A on every smoothed level (P = D, or the
        level's star), lmin / lmax from :func:`jacobi_lanczos_bounds` with a right-hand side seeded by ``seed``."""
        a, b_, c, d_ = esteig
        rng = np.random.default_rng(seed)
        for l in range(1, len(self.spaces)):
            W = self.spaces[l]
            shape = (W.node_count, W.cdim) if W.cdim > 1 else (W.node_count,)
            rhs = W.dat(rng.standard_normal(shape))
            for bc in self.bcs[l]:
                bc.zero(rhs)
            star = self.stars[l]
            lmin, lmax = jacobi_lanczos_bounds(self.ops[l], self.invdiag[l], rhs, esteig_steps,
                                               M=None if star is None else star.apply)
            self.bounds[l] = (a * lmin + b_ * lmax, c * lmin + d_ * lmax)

    def _smooth(self, l, b, x):
        if self.smoother == "richardson":
            return super()._smooth(l, b, x)
        # one action and one fused vector pass per iteration
        from . import _lib
        L = _lib.lib()
        A, w = self.ops[l], self._work[l]
        n = b._data.size
        if self.stars[l] is not None:
            # z = P^-1 (b - A x); d = c_d d + c_z z; x += d
            for cd, cz in chebyshev_coefficients(*self.bounds[l], self.nu):
                A.mult(x, w["t"])
                _lib.check(L.fdb_vec_aypx(n, -1.0, b.device_ptr, w["t"].device_ptr))
                _touched(w["t"])
                self.stars[l].apply(w["t"], w["s"])
                _lib.check(L.fdb_vec_chebyshev(n, cd, cz, w["s"].device_ptr, w["zero"].device_ptr,
                                               w["one"].device_ptr, w["d"].device_ptr, x.device_ptr))
                _touched(w["d"], x)
            return
        for cd, cz in chebyshev_coefficients(*self.bounds[l], self.nu):
            A.mult(x, w["t"])
            _lib.check(L.fdb_vec_chebyshev(n, cd, cz, b.device_ptr, w["t"].device_ptr, self.invdiag[l].device_ptr,
                                           w["d"].device_ptr, x.device_ptr))
            _touched(w["d"], x)

    def _coarse_solve(self, b, x):
        from . import _lib
        from .assemble import cg
        if self.coarse_mg is not None:
            self.coarse_mg.apply(self._coarse_top, b, x)
        elif self.coarse_pc == "none":
            cg(self.ops[0], b, x, rtol=self.coarse_rtol, maxit=self.coarse_maxit)
        else:
            L, d, n = _lib.lib(), self.invdiag[0], b._data.size

            def M(r, z):
                _lib.check(L.fdb_vec_pointwise_mult(n, r.device_ptr, d.device_ptr, z.device_ptr))
                _touched(z)
            pcg(self.ops[0], b, x, M, rtol=self.coarse_rtol, maxit=self.coarse_maxit)
        _touched(x)


class PMG(_SmoothedCycle):
    """p-multigrid on one mesh (Firedrake's ``firedrake.PMGPC`` / ``firedrake.P1PC``): the levels are CG spaces of
    falling degree on ``V.mesh`` (:func:`pmg_degrees`), the operators rediscretised on every level, the transfers
    :class:`PTransfer`.  The cycle is :class:`VCycle`'s (``_LevelCycle.apply``); the top level is ``len(ops) - 1``.

    ``make_form(W[, kappa])``: the form on a level space (with the level's coefficient when ``kappa``, a Dat on
    ``V``, is given; each coarser level gets the injection of the next finer one's).  ``bc_domains``: the
    Dirichlet sub-domains, whose rows are zeroed on every level.

    Smoother on the levels above the coarsest: ``smoother`` "chebyshev" (Chebyshev-Jacobi, ``nu`` iterations with
    the bounds ``esteig`` = (a, b, c, d): [a lmin + b lmax, c lmin + d lmax] with lmin, lmax of D^-1 A estimated
    by :func:`jacobi_lanczos_bounds` in ``esteig_steps`` steps from a right-hand side seeded by ``seed``) or "richardson" (damped Jacobi with ``omega``, ``nu`` sweeps).
    ``level_pc`` "jacobi" (the above) or "star": Chebyshev preconditioned by the fast-diagonalisation vertex-star
    relaxation of the level form (:class:`patch.FDMStar`, ``ASMExtrudedStarPC`` under FDMPC), with the bounds of
    P^-1 A; "star" takes scalar :class:`assemble.Form` levels without ``ds`` terms and the "chebyshev" smoother.

    Coarse solve: ``coarse_ksp`` "cg" with ``coarse_pc`` "jacobi" or "none" to ``coarse_rtol`` /
    ``coarse_maxit``, or "preonly" with "mg": one :class:`VCycle` at the coarse degree on ``hierarchy``, whose
    finest mesh must be ``V.mesh`` and whose top space then is this hierarchy's coarse space."""

    def __init__(self, V, make_form, bc_domains=(), coarse_degree=1, halve=True, kappa=None, smoother="chebyshev",
                 nu=2, omega=0.8, esteig=(0.0, 0.1, 0.0, 1.1), esteig_steps=10, coarse_ksp="cg", coarse_pc="jacobi",
                 coarse_rtol=1e-3, coarse_maxit=500, hierarchy=None, allreduce=None, scatter="atomic", seed=0,
                 level_pc="jacobi"):
        from .assemble import DirichletBC, FunctionSpace, assemble
        if getattr(V, "family", "CG") == "NCF":
            raise NotImplementedError("PMG does not take NCF (H(div)) spaces: the only form on NCF is "
                                      "MixedPoisson")
        if getattr(V, "family", "CG") != "CG":
            raise NotImplementedError("PMG takes CG spaces (there is no DQ p-multigrid)")
        if allreduce is not None or V.dof_dset.halo is not None:
            raise NotImplementedError("PMG on a partitioned space is not implemented (multi-GPU p-multigrid)")
        if V.degree <= coarse_degree or coarse_degree < 1:
            raise ValueError(f"PMG: fine degree {V.degree} has nothing to coarsen to degree {coarse_degree}")
        if V.degree > 3:
            raise NotImplementedError(f"PMG: fine degree {V.degree}: the Jacobi smoother needs the diagonal, which "
                                      f"the hand-written kernels give up to degree 3")
        if smoother not in ("chebyshev", "richardson"):
            raise NotImplementedError(f"PMG level smoother {smoother!r}: 'chebyshev' or 'richardson'")
        if level_pc not in ("jacobi", "star") or (level_pc == "star" and smoother != "chebyshev"):
            raise NotImplementedError(f"PMG level pc {level_pc!r} with smoother {smoother!r}: 'jacobi', or 'star' "
                                      f"under 'chebyshev'")
        self.level_pc = level_pc
        if (coarse_ksp, coarse_pc) not in (("cg", "jacobi"), ("cg", "none"), ("preonly", "mg")):
            raise NotImplementedError(f"PMG coarse solve ksp_type {coarse_ksp!r} with pc_type {coarse_pc!r}: cg with "
                                      f"jacobi or none, or preonly with mg")
        self.nu, self.omega, self.smoother = nu, omega, smoother
        self.coarse_ksp, self.coarse_pc = coarse_ksp, coarse_pc
        self.coarse_rtol, self.coarse_maxit = coarse_rtol, coarse_maxit
        self.degrees = pmg_degrees(V.degree, coarse_degree, halve)
        self.coarse_mg = None
        spaces = [FunctionSpace(V.mesh, q, V.cdim) for q in self.degrees[:-1]] + [V]
        self.transfers = [PTransfer(spaces[l], spaces[l + 1], scatter) for l in range(len(spaces) - 1)]
        if kappa is not None:
            kappas = [kappa]
            for T in self.transfers[::-1]:
                kappas.insert(0, T.inject(kappas[0], T.Vc.dat()))
            self.kappas = kappas
        if coarse_pc == "mg":
            # the same mesh object: the coarse space becomes the V-cycle's top space, which PTransfer pairs with the
            # finer PMG levels on V.mesh
            if hierarchy is None or hierarchy[len(hierarchy) - 1] is not V.mesh:
                raise ValueError("PMG coarse pc_type mg needs a mesh hierarchy whose finest mesh is V's mesh")
            self.coarse_mg = VCycle(hierarchy, coarse_degree, make_form, bc_domains, omega=omega,
                                    kappa=None if kappa is None else self.kappas[0], cdim=V.cdim)
            self._coarse_top = len(hierarchy) - 1
            spaces[0] = self.coarse_mg.spaces[-1]     # the same numbering as FunctionSpace(V.mesh, coarse_degree)
            self.transfers[0] = PTransfer(spaces[0], spaces[1], scatter)
        self.spaces = spaces
        self.bcs = [[DirichletBC(W, 0.0, s) for s in bc_domains] for W in spaces]
        self.ops, self.invdiag, self.stars = [], [], [None] * len(spaces)
        for l, W in enumerate(spaces):
            if l == 0 and self.coarse_mg is not None:
                self.ops.append(self.coarse_mg.ops[-1])
                self.invdiag.append(self.coarse_mg.invdiag[-1])
                continue
            f = make_form(W) if kappa is None else make_form(W, self.kappas[l])
            A = assemble(f, bcs=self.bcs[l], mat_type="matfree")
            self.ops.append(A)
            if l > 0 and level_pc == "star":
                from .patch import FDMStar
                self.stars[l] = FDMStar(f, self.bcs[l])
                self.invdiag.append(None)
                continue
            d = A.getDiagonal(W.dat())
            op2.par_loop(reciprocal_kernel(V.cdim), W.node_set, d(op2.RW))
            self.invdiag.append(d)
        self._work = [dict(r=W.dat(), e=W.dat(), t=W.dat(), b=W.dat(), x=W.dat(), d=W.dat()) for W in spaces]
        if level_pc == "star":
            # the fused Chebyshev pass takes the preconditioned residual as its b, with ax = 0 and dinv = 1
            for l in range(1, len(spaces)):
                w = self._work[l]
                w["s"], w["zero"], w["one"] = (spaces[l].dat(np.full(spaces[l].node_count, v)) for v in (0.0, 0.0, 1.0))
        self.top = len(spaces) - 1
        # Chebyshev bounds of D^-1 A on every smoothed level
        self.bounds = [None] * len(spaces)
        if smoother == "chebyshev":
            self._estimate_bounds(esteig, esteig_steps, seed)


# ---------------------------------------------------------- GTMG for the trace system
def trace_transfer_kernels(k):
    """(prolong, restrict): the transfers between CG1 and the HDiv-trace space of degree k - 1 (k = 2, 3) as plain C
    on the generic wrapper path, the statement that csrc/trace_transfer_hex.cu is checked against and the baseline it
    is measured against.  prolong(lambda WRITE, c READ): trace dof (face 2d + s, GL indices t0, t1 along the
    tangential axes e0 < e1) = sum over the face's 4 vertices of P1[t0][a_e0] P1[t1][a_e1] c; restrict(c INC, lambda
    READ, w READ) adds the transpose applied to w * lambda."""
    if k not in (2, 3):
        raise NotImplementedError(f"trace transfers: k = {k}: the hybridised trace spaces are k = 2, 3")
    table = f"static const double P1[{k}][2] = {_table(op2.trace_transfer_table(k))};\n"
    loop = f"""
    for (int d = 0; d < 3; ++d) {{
        const int e0 = d == 0 ? 1 : 0, e1 = d == 2 ? 1 : 2;
        for (int s = 0; s < 2; ++s)
            for (int t0 = 0; t0 < {k}; ++t0)
                for (int t1 = 0; t1 < {k}; ++t1) {{
                    const int t = (2 * d + s) * {k * k} + t0 * {k} + t1;
                    BODY
                }}
    }}"""
    vert = ("const int lv = (s << (2 - d)) | ((b >> 1) << (2 - e0)) | ((b & 1) << (2 - e1));\n"
            "                        const double p = P1[t0][b >> 1] * P1[t1][b & 1];")
    pro = loop.replace("BODY", f"""double v = 0.0;
                    for (int b = 0; b < 4; ++b) {{
                        {vert}
                        v += p * c[lv];
                    }}
                    lam[t] = v;""")
    res = loop.replace("BODY", f"""const double wl = w[t] * lam[t];
                    for (int b = 0; b < 4; ++b) {{
                        {vert}
                        c[lv] += p * wl;
                    }}""")
    return (CStringKernel(table + f"static void trace_prolong(double *lam, const double *c)\n{{{pro}\n}}\n",
                          "trace_prolong"),
            CStringKernel(table + f"static void trace_restrict(double *c, const double *lam, const double *w)\n"
                                  f"{{{res}\n}}\n", "trace_restrict"))


class TraceTransfer:
    """prolong / restrict between CG1 (``Vc``, ``FunctionSpace(mesh, 1)`` by default) and the HDiv-trace space of a
    :class:`assemble.HybridizationPC`, with :class:`TransferManager`'s interface, on the hand-written kernels of
    csrc/trace_transfer_hex.cu (forms "trace_prolong", "trace_restrict").  prolong is lambda = P c, the trilinear
    interpolant of the vertex values at every trace dof's face point; restrict is c = P^T lambda (exactly: every trace
    dof is weighted by 1 / the number of cells holding it).  ``scatter``: "atomic" or "coloured" (bit-reproducible)
    for the restriction.  ``prolong_generic`` / ``restrict_generic`` run :func:`trace_transfer_kernels` on the generic
    wrapper path."""

    def __init__(self, pc, Vc=None, scatter="atomic"):
        from .assemble import FunctionSpace
        S = pc.form.Sigma
        if Vc is None:
            Vc = FunctionSpace(S.mesh, 1)
        if getattr(Vc, "family", "CG") != "CG" or Vc.degree != 1 or Vc.cdim != 1 or Vc.mesh is not S.mesh:
            raise ValueError("TraceTransfer: the coarse space is scalar CG1 on the hybridised problem's mesh")
        if Vc.dof_dset.halo is not None:
            raise NotImplementedError("TraceTransfer: partitioned spaces are not supported")
        self.pc, self.Vc, self.Vf, self.scatter = pc, Vc, pc.trace, scatter
        self.k = S.degree
        self.cell_set = S.cell_set
        self.cmap = op2.Map(S.cell_set, Vc.node_set, 8, Vc.V.cell_node_map, offset=Vc.V.offset, name="trace_cg1")
        self.tmap = pc.trace_map
        counts = np.bincount(pc.trace.V.full_cell_node_list().ravel(), minlength=pc.trace.node_count)
        self.weight = pc.trace.dat(1.0 / counts)
        kw = dict(degree=self.k - 1, coarse_degree=1)
        self._gk = {f: op2.GlobalKernel(op2.Kernel(f, **kw), maps, extruded=True,
                                        scatter=scatter if f == "trace_restrict" else "atomic")
                    for f, maps in (("trace_prolong", [self.tmap, self.cmap]),
                                    ("trace_restrict", [self.cmap, self.tmap]))}
        self._generic = None

    def prolong(self, coarse: op2.Dat, fine: op2.Dat):
        op2.Parloop(self._gk["trace_prolong"], self.cell_set, [fine(op2.WRITE, self.tmap),
                                                               coarse(op2.READ, self.cmap)])()
        return fine

    def restrict(self, fine_dual: op2.Dat, coarse_dual: op2.Dat):
        coarse_dual.zero()
        coarse_dual.device_ptr                      # materialise the zero on the device
        op2.Parloop(self._gk["trace_restrict"], self.cell_set,
                    [coarse_dual(op2.INC, self.cmap), fine_dual(op2.READ, self.tmap),
                     self.weight(op2.READ, self.tmap)])()
        return coarse_dual

    def prolong_generic(self, coarse: op2.Dat, fine: op2.Dat):
        if self._generic is None:
            self._generic = trace_transfer_kernels(self.k)
        op2.par_loop(self._generic[0], self.cell_set, fine(op2.WRITE, self.tmap), coarse(op2.READ, self.cmap))
        return fine

    def restrict_generic(self, fine_dual: op2.Dat, coarse_dual: op2.Dat):
        if self._generic is None:
            self._generic = trace_transfer_kernels(self.k)
        coarse_dual.zero()
        op2.par_loop(self._generic[1], self.cell_set, coarse_dual(op2.INC, self.cmap), fine_dual(op2.READ, self.tmap),
                     self.weight(op2.READ, self.tmap))
        return coarse_dual


class _TraceNatural:
    """The trace level's "boundary condition": zero the natural-condition faces' multipliers (lambda = 0 there)."""

    def __init__(self, pc):
        self.pc = pc

    def zero(self, d):
        d.zero(self.pc._natural)


class GTMG(_SmoothedCycle):
    """Gopalakrishnan and Tan's non-nested two-level cycle for the trace system H lambda = r of an
    :class:`assemble.HybridizationPC` (Firedrake's ``firedrake.GTMGPC``).  Level 1 is the trace space: operator
    ``pc.mat``, Jacobi diagonal ``pc.diagonal_inverse()``, its natural-condition faces held at zero.  Level 0 is CG1 on
    the same mesh with the rediscretised Laplacian ``Form(P1, 1/alpha, 0.0)`` and Dirichlet conditions on the
    natural sub-domains; the transfers are :class:`TraceTransfer`.  For an affine p, (P p)^T H (P p) = p^T A p /
    alpha: the local problem with affine trace data has the constant flux grad(lambda)/alpha as its exact solution,
    so this coarse operator needs no fitted scale.

    Unlike Firedrake, the engine builds the coarse space and operator itself: no ``appctx`` callbacks
    (``get_coarse_space``, ``get_coarse_operator``, ``coarse_space_bcs``) are read.

    Smoothing, bounds and coarse solves are :class:`PMG`'s: ``smoother`` "chebyshev" (``nu`` iterations, bounds
    ``esteig`` of D^-1 H from ``esteig_steps`` Lanczos steps) or "richardson" (``omega``); ``coarse_ksp`` /
    ``coarse_pc`` "cg" with "jacobi" or "none" to ``coarse_rtol`` / ``coarse_maxit``, or "preonly" with "mg": one
    :class:`VCycle` on ``hierarchy``, whose finest mesh must be the problem's.  ``nullspace``: flux conditions on the
    whole boundary (H 1 = 0, P 1 = 1): the coarse problem is the singular Neumann Laplacian, and the plain mean of its
    right-hand side is removed so that it stays consistent; the caller's CG projects the preconditioned vector."""

    def __init__(self, pc, nullspace=False, smoother="chebyshev", nu=2, omega=0.8, esteig=(0.0, 0.1, 0.0, 1.1),
                 esteig_steps=10, coarse_ksp="cg", coarse_pc="jacobi", coarse_rtol=1e-3, coarse_maxit=500,
                 hierarchy=None, scatter="atomic", seed=0):
        from .assemble import DirichletBC, Form, FunctionSpace, assemble
        if smoother not in ("chebyshev", "richardson"):
            raise NotImplementedError(f"GTMG level smoother {smoother!r}: 'chebyshev' or 'richardson'")
        if (coarse_ksp, coarse_pc) not in (("cg", "jacobi"), ("cg", "none"), ("preonly", "mg")):
            raise NotImplementedError(f"GTMG coarse solve ksp_type {coarse_ksp!r} with pc_type {coarse_pc!r}: cg with "
                                      f"jacobi or none, or preonly with mg")
        F = pc.form
        mesh = F.Sigma.mesh
        self.nu, self.omega, self.smoother = nu, omega, smoother
        self.coarse_ksp, self.coarse_pc = coarse_ksp, coarse_pc
        self.coarse_rtol, self.coarse_maxit = coarse_rtol, coarse_maxit
        self.nullspace = nullspace
        natural = pc.natural_sub_domains

        def make_form(V):
            return Form(V, 1.0 / F.alpha, 0.0)

        self.coarse_mg = None
        if coarse_pc == "mg":
            if hierarchy is None or hierarchy[len(hierarchy) - 1] is not mesh:
                raise ValueError("GTMG coarse pc_type mg needs a mesh hierarchy whose finest mesh is the hybridised "
                                 "problem's mesh")
            self.coarse_mg = VCycle(hierarchy, 1, make_form, natural, omega=omega)
            self._coarse_top = len(hierarchy) - 1
            V1 = self.coarse_mg.spaces[-1]
            bcs0 = self.coarse_mg.bcs[-1]
            A0, d0 = self.coarse_mg.ops[-1], self.coarse_mg.invdiag[-1]
        else:
            V1 = FunctionSpace(mesh, 1)
            bcs0 = [DirichletBC(V1, 0.0, s) for s in natural]
            A0 = assemble(make_form(V1), bcs=bcs0, mat_type="matfree")
            d0 = A0.getDiagonal(V1.dat())
            op2.par_loop(reciprocal_kernel(1), V1.node_set, d0(op2.RW))
        self.pc = pc
        self.spaces = [V1, pc.trace]
        self.bcs = [bcs0, [_TraceNatural(pc)]]
        self.transfers = [TraceTransfer(pc, V1, scatter)]
        self.ops = [A0, pc.mat]
        self.invdiag = [d0, pc.diagonal_inverse()]
        self.stars = [None, None]
        self._work = [dict(r=W.dat(), e=W.dat(), t=W.dat(), b=W.dat(), x=W.dat(), d=W.dat()) for W in self.spaces]
        self._ones = V1.dat(np.ones(V1.node_count)) if nullspace else None
        self.top = 1
        self.bounds = [None, None]
        if smoother == "chebyshev":
            self._estimate_bounds(esteig, esteig_steps, seed)

    def _coarse_solve(self, b, x):
        if self.nullspace:
            b.axpy(-b.inner(self._ones) / b._data.size, self._ones)
        super()._coarse_solve(b, x)

    def __call__(self, r, z):
        """z = one cycle applied to r, from z = 0."""
        z.zero()
        z.device_ptr
        return self.apply(self.top, r, z)
