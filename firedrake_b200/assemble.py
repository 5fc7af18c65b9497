"""The assembly surface: ``assemble()`` for the supported forms, Dirichlet
conditions, and the matrix-free operator context.

Mirrors (same names / call protocol, thin Python over the engine):

* ``firedrake.assemble.assemble`` for 1-forms (``OneFormAssembler``:
  zero tensor -> parloops -> ``bc.zero``; firedrake/assemble.py:1197-1293) and
  2-forms (``ExplicitMatrixAssembler``: sparsity + Mat allocation, parloop with
  BC-masked lgmaps, unit diagonal on BC rows; :1296-1307, 1377-1409, 1484-1525)
* ``firedrake.bcs.DirichletBC.zero/set/apply`` (firedrake/bcs.py:192-221, 404-457)
* ``firedrake.matrix_free.operators.ImplicitMatrixContext`` (operators.py:74-242)

Forms are described by :class:`Form` (the Helmholtz family on a
:class:`FunctionSpace`), :class:`NonlinearDiffusion`, :class:`Elasticity` (linear elasticity on a
vector space) and :class:`HyperElasticity` (its Neo-Hookean counterpart) instead of UFL: UFL/TSFC are not available here, and the
engine keys its kernels on a form descriptor (DESIGN.md section 1).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from . import op2
from .halo import Halo


class FunctionSpace:
    """Scalar/vector CG_p space on an extruded hex mesh, bundling the PyOP2
    objects ``assemble`` needs (node set, cell set, maps, coordinates), i.e.
    what ``V.cell_node_map()``, ``mesh.coordinates.dat`` and friends give in
    Firedrake (firedrake/functionspaceimpl.py:803-812).

    ``family="DQ"``: the scalar discontinuous space DQ_p (p = 1..4) with Gauss-Legendre nodes
    (``mesh.dg_function_space``), for :class:`InteriorPenalty` and the cell forms of :class:`Form`.
    ``element`` is its 1-D element (the kernels' tables); None for CG, whose kernels use the default GLL
    element."""

    def __init__(self, mesh, degree, cdim=1, partition=None, family="CG"):
        self.mesh, self.degree, self.cdim = mesh, degree, cdim
        if family not in ("CG", "DQ"):
            raise ValueError(f"family {family!r}: 'CG' or 'DQ'")
        self.family = family
        self.element = None
        if family == "DQ":
            from .fiat_lite import interval_element
            if cdim != 1:
                raise NotImplementedError("DQ spaces are scalar (vector DQ is not implemented)")
            if partition is not None:
                raise NotImplementedError("partitioned DQ spaces are not implemented: the interior facets on a "
                                          "partition boundary would need both cells")
            self.element = interval_element(degree, variant="gl")
            self.V = V = mesh.dg_function_space(degree)
        else:
            self.V = V = mesh.function_space(degree)
        if partition is not None:
            cell_sizes, node_sizes = partition.cell_sizes, partition.node_sizes
            halo = Halo(partition.halo_lists(V), max_cdim=cdim) if partition.nranks > 1 else None
        else:
            cell_sizes, node_sizes, halo = mesh.num_base_cells, V.node_count, None
        self.cell_set = op2.ExtrudedSet(op2.Set(cell_sizes), mesh.layers)
        # exec-halo partition: a property of the WHOLE distributed set (the last rank holds no
        # exec cells but must follow the same protocol)
        self.cell_set.owner_computes = bool(getattr(partition, "exec_halo", False))
        self.node_set = op2.Set(node_sizes)
        self.dof_dset = op2.DataSet(self.node_set, cdim, halo=halo)
        self.vertex_set = op2.Set(mesh.coord_space.node_count)
        self.cell_node_map = op2.Map(self.cell_set, self.node_set, V.arity, V.cell_node_map,
                                     offset=V.offset)
        self.coord_map = op2.Map(self.cell_set, self.vertex_set, 8, mesh.coord_map,
                                 offset=mesh.coord_offset)
        self.coordinates = op2.Dat(op2.DataSet(self.vertex_set, 3), mesh.coordinates)

    def dat(self, data=None, pinned=False):
        return op2.Dat(self.dof_dset, data, pinned=pinned)

    def vector_dset(self, dim=3):
        """``op2.DataSet(V.node_set, dim)``: ``dim`` values per node of this space (AoS), e.g. the velocity
        of :class:`AdvectionDiffusion` on a scalar space.  On a partitioned space its ghost rows are
        exchanged with the same neighbours as the space's own."""
        if dim == self.cdim:
            return self.dof_dset
        cache = self.__dict__.setdefault("_vector_dsets", {})
        if dim not in cache:
            h = self.dof_dset.halo
            cache[dim] = op2.DataSet(self.node_set, dim,
                                     halo=Halo(h.neighbours, max_cdim=dim) if h is not None else None)
        return cache[dim]

    def cells_are_affine(self):
        """True iff every cell is a parallelepiped (checked on the device, cached per version of
        the coordinate Dat): lets the assembler pick the per-cell-metric kernel variant."""
        import ctypes as C
        from . import _lib
        key = self.coordinates.dat_version
        if getattr(self, "_affine", (None, None))[0] != key:
            off = np.ascontiguousarray(self.mesh.coord_offset, dtype=np.int32)
            res = C.c_int()
            _lib.check(_lib.lib().fdb_cells_are_affine(
                self.coordinates.device_ptr, self.coord_map.device_ptr, off.ctypes.data, 0,
                self.cell_set.total_size, self.mesh.nz, C.byref(res)), "fdb_cells_are_affine")
            self._affine = (key, bool(res.value))
        return self._affine[1]

    @property
    def node_count(self):
        return self.V.node_count

    def boundary_nodes(self, sub_domain):
        return self.V.boundary_nodes(sub_domain)


def _refuse_dq(V, what, why="it is stated on CG spaces only"):
    if getattr(V, "family", "CG") == "DQ":
        raise NotImplementedError(f"{what} does not take DQ spaces: {why}")


def interpolate_q1(V: "FunctionSpace", source: op2.Dat, target: op2.Dat = None):
    """``Function(V).interpolate(w)`` for a Q1 (x) P1 source ``w`` (scalar or
    vector, e.g. the mesh coordinates -> the physical position of every node of
    V): the dual-evaluation parloop of firedrake/interpolation.py:977-1171 with
    WRITE access on the target.  Returns the target Dat (device resident)."""
    from . import _lib
    from .fiat_lite import interval_element
    _refuse_dq(V, "interpolate_q1", "it evaluates at the GLL node positions of CG_p")
    cdim = source.cdim
    if target is None:
        target = op2.Dat(op2.DataSet(V.node_set, cdim))
    if not hasattr(V, "_dev_offsets"):
        V._dev_offsets = (op2.DeviceArray.from_host(np.ascontiguousarray(V.V.offset, dtype=np.int32)),
                          op2.DeviceArray.from_host(np.ascontiguousarray(V.mesh.coord_offset, dtype=np.int32)))
    nodes = np.ascontiguousarray(interval_element(V.degree).nodes, dtype=np.float64)
    _lib.check(_lib.lib().fdb_interpolate_q1(
        target.device_ptr, source.device_ptr, V.cell_node_map.device_ptr, V.coord_map.device_ptr,
        V._dev_offsets[0].ptr, V._dev_offsets[1].ptr, V.cell_set.total_size, V.mesh.nz, V.degree + 1,
        cdim, nodes.ctypes.data), "fdb_interpolate_q1")
    target._device_written()
    return target


def interpolation_kernel(degree, expressions, name="interpolate_expr"):
    """C source of the dual-evaluation kernel of ``Function(V).interpolate(expr(x))`` on
    Q_p (x) P_p with GLL nodes (point evaluation: firedrake/interpolation.py:977-1171
    builds it with tsfc.compile_expression_dual_evaluation, tsfc/driver.py:225-386).
    ``expressions``: one C expression per component in ``x[0], x[1], x[2]`` (the physical
    position of the node, the trilinear image of its reference position) -- the syntax of
    the reference's former ``Expression("sin(x[0])")``.  Arguments: out (WRITE), coords."""
    from .fiat_lite import interval_element
    from .codegen import CStringKernel
    exprs = [expressions] if isinstance(expressions, str) else list(expressions)
    n = degree + 1
    xi = ", ".join(repr(float(v)) for v in interval_element(degree).nodes)
    body = "\n".join(f"        out[i * {len(exprs)} + {c}] = {e};" for c, e in enumerate(exprs))
    code = f"""
static void {name}(double *out, const double *X)
{{
    const double xi[{n}] = {{{xi}}};                 /* 1-D node positions, dof numbering */
    for (int ax = 0; ax < {n}; ++ax)
    for (int ay = 0; ay < {n}; ++ay)
    for (int az = 0; az < {n}; ++az) {{
        const int i = (ax * {n} + ay) * {n} + az;
        double x[3] = {{0.0, 0.0, 0.0}};
        for (int v = 0; v < 8; ++v) {{
            const double w = ((v & 4) ? xi[ax] : 1.0 - xi[ax]) * ((v & 2) ? xi[ay] : 1.0 - xi[ay])
                           * ((v & 1) ? xi[az] : 1.0 - xi[az]);
            for (int c = 0; c < 3; ++c) x[c] += w * X[v * 3 + c];
        }}
{body}
    }}
}}
"""
    return CStringKernel(code, name)


def interpolate(V: "FunctionSpace", expressions, target: op2.Dat = None):
    """``Function(V).interpolate(expr)`` for C expressions of the physical coordinates
    (SURVEY.md section 8f row f2), run as a WRITE parloop through the engine's generic
    wrapper builder.  Nodes shared by several cells are written by each of them with the
    same value, as in the reference's sequential loop."""
    _refuse_dq(V, "interpolate", "it evaluates at the GLL node positions of CG_p")
    exprs = [expressions] if isinstance(expressions, str) else list(expressions)
    if len(exprs) != V.cdim:
        raise ValueError(f"need {V.cdim} expressions for this space, got {len(exprs)}")
    if target is None:
        target = V.dat()
    k = interpolation_kernel(V.degree, exprs)
    op2.par_loop(k, V.cell_set, target(op2.WRITE, V.cell_node_map), V.coordinates(op2.READ, V.coord_map))
    return target


def functional_kernel(degree, measure, facet=None, name=None, integrand="avg"):
    """C source of the 0-form kernels ``f*dx`` and ``f*ds`` on Q_p (x) P_p hexes with
    trilinear geometry (what TSFC emits for a rank-0 form: ``A[0] += w*|J|*f(q)``,
    tsfc/kernel_interface/common.py:139-239; facet kernels get the local facet number
    as ``uint facet[1]``, firedrake_loopy.py:317-381).  Gauss-Legendre p+1 points per
    direction.  ``measure``: "dx" (args: out, coords, f) or "ds" (exterior facet; the
    local facet 2*direction + side is baked in when ``facet`` is given -- the
    extruded ds_b / ds_t kernels -- else read from a 4th argument: ds_v), or "dS" (interior
    facet; ``integrand`` "avg" = avg(f), "jump2" = (f('+') - f('-'))**2; ``facet`` = the pair of
    local facet numbers or None to read uint[2])."""
    from .fiat_lite import interval_element
    from .codegen import CStringKernel
    el = interval_element(degree)
    n = degree + 1
    Bend, _ = el.tabulate([0.0, 1.0])
    tab = lambda a: "{" + ", ".join("{" + ", ".join(repr(float(v)) for v in r) + "}" for r in a) + "}"
    vec = lambda a: "{" + ", ".join(repr(float(v)) for v in a) + "}"
    head = f"""
static const double FB[{n}][{n}] = {tab(el.B)};      /* basis a at Gauss point q: FB[q][a] */
static const double FE[2][{n}] = {tab(Bend)};        /* basis at the interval's ends */
static const double FX[{n}] = {vec(el.xq)};
static const double FW[{n}] = {vec(el.wq)};
/* columns of the Jacobian of the trilinear map at xi: J[c][d] = dx_c / dxi_d */
static inline void q1_jacobian(const double *X, const double *xi, double J[3][3])
{{
    for (int c = 0; c < 3; ++c) for (int d = 0; d < 3; ++d) J[c][d] = 0.0;
    for (int v = 0; v < 8; ++v) {{
        const int b[3] = {{(v >> 2) & 1, (v >> 1) & 1, v & 1}};
        for (int d = 0; d < 3; ++d) {{
            double g = b[d] ? 1.0 : -1.0;
            for (int e = 0; e < 3; ++e) if (e != d) g *= b[e] ? xi[e] : 1.0 - xi[e];
            for (int c = 0; c < 3; ++c) J[c][d] += X[v * 3 + c] * g;
        }}
    }}
}}
"""
    if measure == "dx":
        name = name or "functional_dx"
        code = head + f"""
static void {name}(double *out, const double *X, const double *f)
{{
    for (int qx = 0; qx < {n}; ++qx) for (int qy = 0; qy < {n}; ++qy) for (int qz = 0; qz < {n}; ++qz) {{
        const double xi[3] = {{FX[qx], FX[qy], FX[qz]}};
        double J[3][3], v = 0.0;
        q1_jacobian(X, xi, J);
        const double det = J[0][0] * (J[1][1] * J[2][2] - J[1][2] * J[2][1])
                         - J[0][1] * (J[1][0] * J[2][2] - J[1][2] * J[2][0])
                         + J[0][2] * (J[1][0] * J[2][1] - J[1][1] * J[2][0]);
        for (int a = 0; a < {n}; ++a) for (int b = 0; b < {n}; ++b) for (int c = 0; c < {n}; ++c)
            v += f[(a * {n} + b) * {n} + c] * FB[qx][a] * FB[qy][b] * FB[qz][c];
        out[0] += FW[qx] * FW[qy] * FW[qz] * fabs(det) * v;
    }}
}}
"""
        return CStringKernel(code, name)
    if measure == "dS":
        # interior facets: coefficient and coordinate arrays are doubled, cell '+' then cell '-'
        # (tsfc/kernel_interface/common.py:518-522); local facet numbers uint[2]
        # (firedrake_loopy.py:317-381).  The two cells are conforming and equally oriented, so a
        # quadrature point has the same tangential reference coordinates in both.
        name = name or ("functional_dS" if facet is None else f"functional_dS{facet[0]}{facet[1]}")
        sig = ", const unsigned int *facet" if facet is None else ""
        getp, getm = ("facet[0]", "facet[1]") if facet is None else (str(int(facet[0])), str(int(facet[1])))
        expr = {"avg": "0.5 * (v[0] + v[1])", "jump2": "(v[0] - v[1]) * (v[0] - v[1])"}[integrand]
        code = head + f"""
static void {name}(double *out, const double *X, const double *f{sig})
{{
    const int fac[2] = {{(int)({getp}), (int)({getm})}};
    const int fd = fac[0] / 2, d1 = (fd + 1) % 3, d2 = (fd + 2) % 3;
    for (int q1 = 0; q1 < {n}; ++q1) for (int q2 = 0; q2 < {n}; ++q2) {{
        double xi[3], J[3][3], v[2];
        const double *T[3];
        for (int s = 0; s < 2; ++s) {{                 /* restriction '+' (s = 0) and '-' (s = 1) */
            T[fd] = FE[fac[s] % 2]; T[d1] = FB[q1]; T[d2] = FB[q2];
            v[s] = 0.0;
            for (int a = 0; a < {n}; ++a) for (int b = 0; b < {n}; ++b) for (int c = 0; c < {n}; ++c)
                v[s] += f[s * {n ** 3} + (a * {n} + b) * {n} + c] * T[0][a] * T[1][b] * T[2][c];
        }}
        xi[fd] = (double)(fac[0] % 2); xi[d1] = FX[q1]; xi[d2] = FX[q2];
        q1_jacobian(X, xi, J);                          /* geometry from the '+' cell */
        const double cx = J[1][d1] * J[2][d2] - J[2][d1] * J[1][d2];
        const double cy = J[2][d1] * J[0][d2] - J[0][d1] * J[2][d2];
        const double cz = J[0][d1] * J[1][d2] - J[1][d1] * J[0][d2];
        out[0] += FW[q1] * FW[q2] * sqrt(cx * cx + cy * cy + cz * cz) * ({expr});
    }}
}}
"""
        return CStringKernel(code, name)
    if measure != "ds":
        raise ValueError(f"unknown measure {measure!r}")
    name = name or ("functional_ds" if facet is None else f"functional_ds{facet}")
    sig = "const unsigned int *facet" if facet is None else ""
    get = "facet[0]" if facet is None else str(int(facet))
    code = head + f"""
static void {name}(double *out, const double *X, const double *f{", " + sig if sig else ""})
{{
    const int fd = (int)({get}) / 2, fs = (int)({get}) % 2;     /* normal direction, side */
    const int d1 = (fd + 1) % 3, d2 = (fd + 2) % 3;
    for (int q1 = 0; q1 < {n}; ++q1) for (int q2 = 0; q2 < {n}; ++q2) {{
        double xi[3], J[3][3], v = 0.0;
        const double *T[3];                       /* 1-D basis rows per direction */
        xi[fd] = (double)fs; xi[d1] = FX[q1]; xi[d2] = FX[q2];
        T[fd] = FE[fs]; T[d1] = FB[q1]; T[d2] = FB[q2];
        q1_jacobian(X, xi, J);
        /* surface element |dx/dxi_d1 x dx/dxi_d2| */
        const double cx = J[1][d1] * J[2][d2] - J[2][d1] * J[1][d2];
        const double cy = J[2][d1] * J[0][d2] - J[0][d1] * J[2][d2];
        const double cz = J[0][d1] * J[1][d2] - J[1][d1] * J[0][d2];
        for (int a = 0; a < {n}; ++a) for (int b = 0; b < {n}; ++b) for (int c = 0; c < {n}; ++c)
            v += f[(a * {n} + b) * {n} + c] * T[0][a] * T[1][b] * T[2][c];
        out[0] += FW[q1] * FW[q2] * sqrt(cx * cx + cy * cy + cz * cz) * v;
    }}
}}
"""
    return CStringKernel(code, name)


def variable_coefficient_kernel(degree, beta=0.0, name="varcoef_action"):
    """C source of the 1-form ``action(inner(kappa*grad(u), grad(v))*dx + beta*inner(u, v)*dx, u)``
    with a COEFFICIENT FIELD kappa in the same Q_p (x) P_p space -- a form outside the hand-written
    set, written the way TSFC's spectral mode would (sum factorisation, tsfc/spectral.py:24-191;
    coefficients are tabulated like arguments, tsfc/fem.py:710-804) and run through the generic
    wrapper builder.  Arguments: y (INC), coords, u, kappa."""
    from .fiat_lite import interval_element
    from .codegen import CStringKernel
    el = interval_element(degree)
    n = degree + 1
    tab = lambda a: "{" + ", ".join("{" + ", ".join(repr(float(v)) for v in r) + "}" for r in a) + "}"
    vec = lambda a: "{" + ", ".join(repr(float(v)) for v in a) + "}"
    code = f"""
#define VN {n}
static const double VB[VN][VN] = {tab(el.B)};      /* VB[q][a] */
static const double VD[VN][VN] = {tab(el.D)};      /* VD[q][a] */
static const double VX[VN] = {vec(el.xq)};
static const double VW[VN] = {vec(el.wq)};
/* out = (T applied along direction dir) in;  tr = 0: out[q] = sum_a T[q][a] in[a];  tr = 1: transpose */
static inline void vc_apply(const double T[VN][VN], int dir, int tr, const double *in, double *out)
{{
    const int st = dir == 0 ? VN * VN : (dir == 1 ? VN : 1);
    for (int i = 0; i < VN * VN * VN; ++i) {{
        const int k = (i / st) % VN, base = i - k * st;
        double s = 0.0;
        for (int a = 0; a < VN; ++a) s += (tr ? T[a][k] : T[k][a]) * in[base + a * st];
        out[i] = s;
    }}
}}
static inline void vc_tensor(const double (*T0)[VN], const double (*T1)[VN], const double (*T2)[VN], int tr,
                             const double *in, double *out)
{{
    double t1[VN * VN * VN], t2[VN * VN * VN];
    vc_apply(T0, 0, tr, in, t1);
    vc_apply(T1, 1, tr, t1, t2);
    vc_apply(T2, 2, tr, t2, out);
}}
static void {name}(double *y, const double *X, const double *u, const double *kappa)
{{
    double U[VN * VN * VN], G[3][VN * VN * VN], K[VN * VN * VN], t[VN * VN * VN];
    vc_tensor(VB, VB, VB, 0, u, U);
    vc_tensor(VD, VB, VB, 0, u, G[0]);
    vc_tensor(VB, VD, VB, 0, u, G[1]);
    vc_tensor(VB, VB, VD, 0, u, G[2]);
    vc_tensor(VB, VB, VB, 0, kappa, K);
    for (int qx = 0; qx < VN; ++qx) for (int qy = 0; qy < VN; ++qy) for (int qz = 0; qz < VN; ++qz) {{
        const int q = (qx * VN + qy) * VN + qz;
        const double xi[3] = {{VX[qx], VX[qy], VX[qz]}};
        double J[3][3] = {{{{0}}}};
        for (int v = 0; v < 8; ++v) {{
            const int b[3] = {{(v >> 2) & 1, (v >> 1) & 1, v & 1}};
            for (int d = 0; d < 3; ++d) {{
                double g = b[d] ? 1.0 : -1.0;
                for (int e = 0; e < 3; ++e) if (e != d) g *= b[e] ? xi[e] : 1.0 - xi[e];
                for (int c = 0; c < 3; ++c) J[c][d] += X[v * 3 + c] * g;
            }}
        }}
        double R[3][3];                              /* cofactor rows: R[k] . J[:, m] = det * delta_km */
        R[0][0] = J[1][1] * J[2][2] - J[2][1] * J[1][2]; R[0][1] = J[2][1] * J[0][2] - J[0][1] * J[2][2];
        R[0][2] = J[0][1] * J[1][2] - J[1][1] * J[0][2];
        R[1][0] = J[1][2] * J[2][0] - J[2][2] * J[1][0]; R[1][1] = J[2][2] * J[0][0] - J[0][2] * J[2][0];
        R[1][2] = J[0][2] * J[1][0] - J[1][2] * J[0][0];
        R[2][0] = J[1][0] * J[2][1] - J[2][0] * J[1][1]; R[2][1] = J[2][0] * J[0][1] - J[0][0] * J[2][1];
        R[2][2] = J[0][0] * J[1][1] - J[1][0] * J[0][1];
        const double det = J[0][0] * R[0][0] + J[1][0] * R[0][1] + J[2][0] * R[0][2];
        const double w = VW[qx] * VW[qy] * VW[qz];
        double h[3], f[3];
        for (int c = 0; c < 3; ++c) h[c] = R[0][c] * G[0][q] + R[1][c] * G[1][q] + R[2][c] * G[2][q];
        for (int k = 0; k < 3; ++k)
            f[k] = K[q] * w / fabs(det) * (R[k][0] * h[0] + R[k][1] * h[1] + R[k][2] * h[2]);
        G[0][q] = f[0]; G[1][q] = f[1]; G[2][q] = f[2];
        U[q] *= {float(beta)!r} * w * fabs(det);
    }}
    vc_tensor(VD, VB, VB, 1, G[0], t);  for (int i = 0; i < VN * VN * VN; ++i) y[i] += t[i];
    vc_tensor(VB, VD, VB, 1, G[1], t);  for (int i = 0; i < VN * VN * VN; ++i) y[i] += t[i];
    vc_tensor(VB, VB, VD, 1, G[2], t);  for (int i = 0; i < VN * VN * VN; ++i) y[i] += t[i];
    vc_tensor(VB, VB, VB, 1, U, t);     for (int i = 0; i < VN * VN * VN; ++i) y[i] += t[i];
}}
#undef VN
"""
    return CStringKernel(code, name)


def assemble_variable_coefficient(V: "FunctionSpace", kappa: op2.Dat, u: op2.Dat, beta=0.0, tensor=None, bcs=()):
    """``assemble(action(inner(kappa*grad(u), grad(v))*dx + beta*inner(u, v)*dx, u))`` for a scalar
    coefficient field ``kappa`` in V (generic path)."""
    if V.cdim != 1:
        raise NotImplementedError("scalar spaces only")
    if tensor is None:
        tensor = V.dat()
    tensor.zero()
    tensor.device_ptr
    op2.par_loop(variable_coefficient_kernel(V.degree, beta), V.cell_set, tensor(op2.INC, V.cell_node_map),
                 V.coordinates(op2.READ, V.coord_map), u(op2.READ, V.cell_node_map),
                 kappa(op2.READ, V.cell_node_map))
    for bc in bcs:
        bc.zero(tensor)
    return tensor


def _vector_hex_tables(degree):
    """C preamble of the generic-path vector (3 component) hex kernels: the 1-D tables of the Q_p (x) P_p
    element and the sum-factorised tensor contraction ``el_tensor``."""
    from .fiat_lite import interval_element
    el = interval_element(degree)
    n = degree + 1
    tab = lambda a: "{" + ", ".join("{" + ", ".join(repr(float(v)) for v in r) + "}" for r in a) + "}"
    vec = lambda a: "{" + ", ".join(repr(float(v)) for v in a) + "}"
    return f"""
#define EN {n}
#define END (EN * EN * EN)
static const double EB[EN][EN] = {tab(el.B)};      /* EB[q][a] */
static const double ED[EN][EN] = {tab(el.D)};      /* ED[q][a] */
static const double EX[EN] = {vec(el.xq)};
static const double EW[EN] = {vec(el.wq)};
/* out = (T applied along direction dir) in;  tr = 0: out[q] = sum_a T[q][a] in[a];  tr = 1: transpose */
static inline void el_apply(const double T[EN][EN], int dir, int tr, const double *in, double *out)
{{
    const int st = dir == 0 ? EN * EN : (dir == 1 ? EN : 1);
    for (int i = 0; i < END; ++i) {{
        const int k = (i / st) % EN, base = i - k * st;
        double s = 0.0;
        for (int a = 0; a < EN; ++a) s += (tr ? T[a][k] : T[k][a]) * in[base + a * st];
        out[i] = s;
    }}
}}
static inline void el_tensor(const double (*T0)[EN], const double (*T1)[EN], const double (*T2)[EN], int tr,
                             const double *in, double *out)
{{
    double t1[END], t2[END];
    el_apply(T0, 0, tr, in, t1);
    el_apply(T1, 1, tr, t1, t2);
    el_apply(T2, 2, tr, t2, out);
}}
"""


def elasticity_kernel(degree, mu, lmbda, beta=0.0, name="elasticity_action"):
    """C source of the 1-form ``action(inner(sigma(u), grad(v))*dx + beta*inner(u, v)*dx, u)`` of linear
    elasticity, ``sigma(u) = 2*mu*sym(grad(u)) + lmbda*tr(sym(grad(u)))*Identity(3)``, on the vector
    Q_p (x) P_p space (3 components, AoS), written the way TSFC's spectral mode would and run through the
    generic wrapper builder: the independent statement of the hand-written FDB_FORM_ELASTICITY kernel.
    Arguments: y (INC), coords, u."""
    from .codegen import CStringKernel
    code = _vector_hex_tables(degree) + f"""static void {name}(double *y, const double *X, const double *u)
{{
    double U[3][END], G[3][3][END], c[END], t[END];
    for (int d = 0; d < 3; ++d) {{
        for (int i = 0; i < END; ++i) c[i] = u[i * 3 + d];
        el_tensor(EB, EB, EB, 0, c, U[d]);
        el_tensor(ED, EB, EB, 0, c, G[d][0]);
        el_tensor(EB, ED, EB, 0, c, G[d][1]);
        el_tensor(EB, EB, ED, 0, c, G[d][2]);
    }}
    for (int qx = 0; qx < EN; ++qx) for (int qy = 0; qy < EN; ++qy) for (int qz = 0; qz < EN; ++qz) {{
        const int q = (qx * EN + qy) * EN + qz;
        const double xi[3] = {{EX[qx], EX[qy], EX[qz]}};
        double J[3][3] = {{{{0}}}};
        for (int v = 0; v < 8; ++v) {{
            const int b[3] = {{(v >> 2) & 1, (v >> 1) & 1, v & 1}};
            for (int r = 0; r < 3; ++r) {{
                double g = b[r] ? 1.0 : -1.0;
                for (int e = 0; e < 3; ++e) if (e != r) g *= b[e] ? xi[e] : 1.0 - xi[e];
                for (int k = 0; k < 3; ++k) J[k][r] += X[v * 3 + k] * g;
            }}
        }}
        /* Jinv[m][k] = dxi_m/dx_k */
        const double det = J[0][0] * (J[1][1] * J[2][2] - J[1][2] * J[2][1])
                         - J[0][1] * (J[1][0] * J[2][2] - J[1][2] * J[2][0])
                         + J[0][2] * (J[1][0] * J[2][1] - J[1][1] * J[2][0]);
        double Jinv[3][3];
        Jinv[0][0] = (J[1][1] * J[2][2] - J[1][2] * J[2][1]) / det;
        Jinv[0][1] = (J[0][2] * J[2][1] - J[0][1] * J[2][2]) / det;
        Jinv[0][2] = (J[0][1] * J[1][2] - J[0][2] * J[1][1]) / det;
        Jinv[1][0] = (J[1][2] * J[2][0] - J[1][0] * J[2][2]) / det;
        Jinv[1][1] = (J[0][0] * J[2][2] - J[0][2] * J[2][0]) / det;
        Jinv[1][2] = (J[0][2] * J[1][0] - J[0][0] * J[1][2]) / det;
        Jinv[2][0] = (J[1][0] * J[2][1] - J[1][1] * J[2][0]) / det;
        Jinv[2][1] = (J[0][1] * J[2][0] - J[0][0] * J[2][1]) / det;
        Jinv[2][2] = (J[0][0] * J[1][1] - J[0][1] * J[1][0]) / det;
        const double wd = EW[qx] * EW[qy] * EW[qz] * fabs(det);
        double Gp[3][3], S[3][3];
        for (int d = 0; d < 3; ++d)
            for (int k = 0; k < 3; ++k)
                Gp[d][k] = G[d][0][q] * Jinv[0][k] + G[d][1][q] * Jinv[1][k] + G[d][2][q] * Jinv[2][k];
        const double tr = Gp[0][0] + Gp[1][1] + Gp[2][2];
        for (int d = 0; d < 3; ++d)
            for (int k = 0; k < 3; ++k)
                S[d][k] = {float(mu)!r} * (Gp[d][k] + Gp[k][d]) + (d == k ? {float(lmbda)!r} * tr : 0.0);
        for (int d = 0; d < 3; ++d) {{
            for (int m = 0; m < 3; ++m)
                G[d][m][q] = wd * (Jinv[m][0] * S[d][0] + Jinv[m][1] * S[d][1] + Jinv[m][2] * S[d][2]);
            U[d][q] *= {float(beta)!r} * wd;
        }}
    }}
    for (int d = 0; d < 3; ++d) {{
        el_tensor(EB, EB, EB, 1, U[d], c);
        el_tensor(ED, EB, EB, 1, G[d][0], t);  for (int i = 0; i < END; ++i) c[i] += t[i];
        el_tensor(EB, ED, EB, 1, G[d][1], t);  for (int i = 0; i < END; ++i) c[i] += t[i];
        el_tensor(EB, EB, ED, 1, G[d][2], t);  for (int i = 0; i < END; ++i) c[i] += t[i];
        for (int i = 0; i < END; ++i) y[i * 3 + d] += c[i];
    }}
}}
#undef END
#undef EN
"""
    return CStringKernel(code, name)


def assemble_elasticity_generic(V: "FunctionSpace", u: op2.Dat, mu, lmbda, beta=0.0, tensor=None):
    """``assemble(action(a, u))`` of linear elasticity through the generic wrapper path
    (:func:`elasticity_kernel`): the cross-check and the baseline of :class:`Elasticity`."""
    if V.cdim != 3:
        raise ValueError("elasticity needs a vector space with 3 components")
    if tensor is None:
        tensor = V.dat()
    tensor.zero()
    tensor.device_ptr
    op2.par_loop(elasticity_kernel(V.degree, mu, lmbda, beta), V.cell_set, tensor(op2.INC, V.cell_node_map),
                 V.coordinates(op2.READ, V.coord_map), u(op2.READ, V.cell_node_map))
    return tensor


def stokes_kernel(degree, mu=1.0, beta=0.0, name="stokes_action"):
    """C source of the Stokes action ``mu*inner(grad u, grad v)*dx + beta*inner(u, v)*dx - p*div(v)*dx -
    q*div(u)*dx`` on Taylor-Hood Q_p-Q_(p-1) hexahedra, run through the generic wrapper builder with MixedDat
    arguments: the independent statement of the hand-written FDB_FORM_STOKES kernel.  Arguments: y (INC) and
    up, each the velocity's 3 END values (AoS) followed by the pressure's (EN-1)^3, and the coordinates.
    The pressure is held in an EN^3 block, zero at every dof index EN-1, with its table padded by a zero
    column, so the square contractions of the velocity serve it too."""
    from .codegen import CStringKernel
    from .fiat_lite import interval_element
    if not 2 <= degree <= 4:
        raise NotImplementedError(f"the generic-path Stokes statement covers degrees 2..4, got degree {degree}")
    elq = interval_element(degree - 1, degree + 1)
    n = degree + 1
    bq = [[float(elq.B[q, a]) if a < n - 1 else 0.0 for a in range(n)] for q in range(n)]
    tab = "{" + ", ".join("{" + ", ".join(repr(v) for v in r) + "}" for r in bq) + "}"
    code = _vector_hex_tables(degree) + f"""#define ENP (EN - 1)
static const double EQ[EN][EN] = {tab};      /* EQ[q][a]: pressure basis, zero last column */
static void {name}(double *y, const double *X, const double *up)
{{
    double U[3][END], G[3][3][END], c[END], t[END], P[END], T[END];
    const double *pin = up + 3 * END;
    for (int d = 0; d < 3; ++d) {{
        for (int i = 0; i < END; ++i) c[i] = up[i * 3 + d];
        el_tensor(EB, EB, EB, 0, c, U[d]);
        el_tensor(ED, EB, EB, 0, c, G[d][0]);
        el_tensor(EB, ED, EB, 0, c, G[d][1]);
        el_tensor(EB, EB, ED, 0, c, G[d][2]);
    }}
    for (int i = 0; i < END; ++i) {{
        const int a = i / (EN * EN), b = (i / EN) % EN, e = i % EN;
        c[i] = (a < ENP && b < ENP && e < ENP) ? pin[(a * ENP + b) * ENP + e] : 0.0;
    }}
    el_tensor(EQ, EQ, EQ, 0, c, P);
    for (int qx = 0; qx < EN; ++qx) for (int qy = 0; qy < EN; ++qy) for (int qz = 0; qz < EN; ++qz) {{
        const int q = (qx * EN + qy) * EN + qz;
        const double xi[3] = {{EX[qx], EX[qy], EX[qz]}};
        double J[3][3] = {{{{0}}}};
        for (int v = 0; v < 8; ++v) {{
            const int b[3] = {{(v >> 2) & 1, (v >> 1) & 1, v & 1}};
            for (int r = 0; r < 3; ++r) {{
                double g = b[r] ? 1.0 : -1.0;
                for (int e = 0; e < 3; ++e) if (e != r) g *= b[e] ? xi[e] : 1.0 - xi[e];
                for (int k = 0; k < 3; ++k) J[k][r] += X[v * 3 + k] * g;
            }}
        }}
        const double det = J[0][0] * (J[1][1] * J[2][2] - J[1][2] * J[2][1])
                         - J[0][1] * (J[1][0] * J[2][2] - J[1][2] * J[2][0])
                         + J[0][2] * (J[1][0] * J[2][1] - J[1][1] * J[2][0]);
        double Jinv[3][3];
        Jinv[0][0] = (J[1][1] * J[2][2] - J[1][2] * J[2][1]) / det;
        Jinv[0][1] = (J[0][2] * J[2][1] - J[0][1] * J[2][2]) / det;
        Jinv[0][2] = (J[0][1] * J[1][2] - J[0][2] * J[1][1]) / det;
        Jinv[1][0] = (J[1][2] * J[2][0] - J[1][0] * J[2][2]) / det;
        Jinv[1][1] = (J[0][0] * J[2][2] - J[0][2] * J[2][0]) / det;
        Jinv[1][2] = (J[0][2] * J[1][0] - J[0][0] * J[1][2]) / det;
        Jinv[2][0] = (J[1][0] * J[2][1] - J[1][1] * J[2][0]) / det;
        Jinv[2][1] = (J[0][1] * J[2][0] - J[0][0] * J[2][1]) / det;
        Jinv[2][2] = (J[0][0] * J[1][1] - J[0][1] * J[1][0]) / det;
        const double wd = EW[qx] * EW[qy] * EW[qz] * fabs(det);
        double Gp[3][3], S[3][3];
        for (int d = 0; d < 3; ++d)
            for (int k = 0; k < 3; ++k)
                Gp[d][k] = G[d][0][q] * Jinv[0][k] + G[d][1][q] * Jinv[1][k] + G[d][2][q] * Jinv[2][k];
        for (int d = 0; d < 3; ++d)
            for (int k = 0; k < 3; ++k)
                S[d][k] = {float(mu)!r} * Gp[d][k] - (d == k ? P[q] : 0.0);
        for (int d = 0; d < 3; ++d) {{
            for (int m = 0; m < 3; ++m)
                G[d][m][q] = wd * (Jinv[m][0] * S[d][0] + Jinv[m][1] * S[d][1] + Jinv[m][2] * S[d][2]);
            U[d][q] *= {float(beta)!r} * wd;
        }}
        T[q] = -wd * (Gp[0][0] + Gp[1][1] + Gp[2][2]);
    }}
    for (int d = 0; d < 3; ++d) {{
        el_tensor(EB, EB, EB, 1, U[d], c);
        el_tensor(ED, EB, EB, 1, G[d][0], t);  for (int i = 0; i < END; ++i) c[i] += t[i];
        el_tensor(EB, ED, EB, 1, G[d][1], t);  for (int i = 0; i < END; ++i) c[i] += t[i];
        el_tensor(EB, EB, ED, 1, G[d][2], t);  for (int i = 0; i < END; ++i) c[i] += t[i];
        for (int i = 0; i < END; ++i) y[i * 3 + d] += c[i];
    }}
    el_tensor(EQ, EQ, EQ, 1, T, c);
    for (int a = 0; a < ENP; ++a) for (int b = 0; b < ENP; ++b) for (int e = 0; e < ENP; ++e)
        y[3 * END + (a * ENP + b) * ENP + e] += c[(a * EN + b) * EN + e];
}}
#undef ENP
#undef END
#undef EN
"""
    return CStringKernel(code, name)


def assemble_stokes_generic(F: "Stokes", up: op2.MixedDat, tensor=None):
    """``assemble(action(a, up))`` of :class:`Stokes` through the generic wrapper path (:func:`stokes_kernel`,
    MixedDat arguments over the velocity and pressure maps): the cross-check and the baseline of the
    hand-written kernel."""
    V = F.V
    if tensor is None:
        tensor = F.dat()
    tensor.zero()
    for d in tensor:
        d.device_ptr
    mm = op2.MixedMap([V.cell_node_map, F.pressure_map])
    op2.par_loop(stokes_kernel(V.degree, F.mu, F.beta), V.cell_set, tensor(op2.INC, mm),
                 V.coordinates(op2.READ, V.coord_map), up(op2.READ, mm))
    return tensor


def navier_stokes_kernel(degree, nu=1.0, beta=0.0, jacobian=False, name=None):
    """C source of the steady Navier-Stokes residual ``nu*inner(grad u, grad v)*dx + beta*inner(u, v)*dx +
    inner(dot(grad u, u), v)*dx - p*div(v)*dx - q*div(u)*dx`` on Taylor-Hood Q_p-Q_(p-1) hexahedra (arguments: y
    (INC) and up as in :func:`stokes_kernel`, and the coordinates), or with ``jacobian`` of its Gateaux
    derivative's action at u on (w, r), the Stokes action on (w, r) plus ``inner(dot(grad w, u), v)*dx +
    inner(dot(grad u, w), v)*dx`` (arguments: y (INC), coords, wr, u with u the velocity's 3 END values).  The
    independent statement of the hand-written FDB_FORM_NAVIER_STOKES[_JACOBIAN] kernels, run through the
    generic wrapper builder."""
    from .codegen import CStringKernel
    from .fiat_lite import interval_element
    if not 2 <= degree <= 4:
        raise NotImplementedError(f"the generic-path Navier-Stokes statement covers degrees 2..4, got degree {degree}")
    if name is None:
        name = "navier_stokes_jacobian_action" if jacobian else "navier_stokes_residual"
    elq = interval_element(degree - 1, degree + 1)
    n = degree + 1
    bq = [[float(elq.B[q, a]) if a < n - 1 else 0.0 for a in range(n)] for q in range(n)]
    tab = "{" + ", ".join("{" + ", ".join(repr(v) for v in r) + "}" for r in bq) + "}"
    args = "double *y, const double *X, const double *up, const double *u" if jacobian else \
        "double *y, const double *X, const double *up"
    # the linearisation velocity's values UL and physical gradient GL at the point: u itself for the residual
    lin = """
        double GL[3][3];
        for (int d = 0; d < 3; ++d)
            for (int k = 0; k < 3; ++k)
                GL[d][k] = GU[d][0][q] * Jinv[0][k] + GU[d][1][q] * Jinv[1][k] + GU[d][2][q] * Jinv[2][k];
        for (int d = 0; d < 3; ++d)
            cv[d] = Gp[d][0] * UL[0][q] + Gp[d][1] * UL[1][q] + Gp[d][2] * UL[2][q]
                  + GL[d][0] * U[0][q] + GL[d][1] * U[1][q] + GL[d][2] * U[2][q];""" if jacobian else """
        for (int d = 0; d < 3; ++d) cv[d] = Gp[d][0] * U[0][q] + Gp[d][1] * U[1][q] + Gp[d][2] * U[2][q];"""
    gather_u = """
        for (int i = 0; i < END; ++i) c[i] = u[i * 3 + d];
        el_tensor(EB, EB, EB, 0, c, UL[d]);
        el_tensor(ED, EB, EB, 0, c, GU[d][0]);
        el_tensor(EB, ED, EB, 0, c, GU[d][1]);
        el_tensor(EB, EB, ED, 0, c, GU[d][2]);""" if jacobian else ""
    decl_u = "double UL[3][END], GU[3][3][END];" if jacobian else ""
    code = _vector_hex_tables(degree) + f"""#define ENP (EN - 1)
static const double EQ[EN][EN] = {tab};      /* EQ[q][a]: pressure basis, zero last column */
static void {name}({args})
{{
    double U[3][END], G[3][3][END], c[END], t[END], P[END], T[END];
    {decl_u}
    const double *pin = up + 3 * END;
    for (int d = 0; d < 3; ++d) {{
        for (int i = 0; i < END; ++i) c[i] = up[i * 3 + d];
        el_tensor(EB, EB, EB, 0, c, U[d]);
        el_tensor(ED, EB, EB, 0, c, G[d][0]);
        el_tensor(EB, ED, EB, 0, c, G[d][1]);
        el_tensor(EB, EB, ED, 0, c, G[d][2]);{gather_u}
    }}
    for (int i = 0; i < END; ++i) {{
        const int a = i / (EN * EN), b = (i / EN) % EN, e = i % EN;
        c[i] = (a < ENP && b < ENP && e < ENP) ? pin[(a * ENP + b) * ENP + e] : 0.0;
    }}
    el_tensor(EQ, EQ, EQ, 0, c, P);
    for (int qx = 0; qx < EN; ++qx) for (int qy = 0; qy < EN; ++qy) for (int qz = 0; qz < EN; ++qz) {{
        const int q = (qx * EN + qy) * EN + qz;
        const double xi[3] = {{EX[qx], EX[qy], EX[qz]}};
        double J[3][3] = {{{{0}}}};
        for (int v = 0; v < 8; ++v) {{
            const int b[3] = {{(v >> 2) & 1, (v >> 1) & 1, v & 1}};
            for (int r = 0; r < 3; ++r) {{
                double g = b[r] ? 1.0 : -1.0;
                for (int e = 0; e < 3; ++e) if (e != r) g *= b[e] ? xi[e] : 1.0 - xi[e];
                for (int k = 0; k < 3; ++k) J[k][r] += X[v * 3 + k] * g;
            }}
        }}
        const double det = J[0][0] * (J[1][1] * J[2][2] - J[1][2] * J[2][1])
                         - J[0][1] * (J[1][0] * J[2][2] - J[1][2] * J[2][0])
                         + J[0][2] * (J[1][0] * J[2][1] - J[1][1] * J[2][0]);
        double Jinv[3][3];
        Jinv[0][0] = (J[1][1] * J[2][2] - J[1][2] * J[2][1]) / det;
        Jinv[0][1] = (J[0][2] * J[2][1] - J[0][1] * J[2][2]) / det;
        Jinv[0][2] = (J[0][1] * J[1][2] - J[0][2] * J[1][1]) / det;
        Jinv[1][0] = (J[1][2] * J[2][0] - J[1][0] * J[2][2]) / det;
        Jinv[1][1] = (J[0][0] * J[2][2] - J[0][2] * J[2][0]) / det;
        Jinv[1][2] = (J[0][2] * J[1][0] - J[0][0] * J[1][2]) / det;
        Jinv[2][0] = (J[1][0] * J[2][1] - J[1][1] * J[2][0]) / det;
        Jinv[2][1] = (J[0][1] * J[2][0] - J[0][0] * J[2][1]) / det;
        Jinv[2][2] = (J[0][0] * J[1][1] - J[0][1] * J[1][0]) / det;
        const double wd = EW[qx] * EW[qy] * EW[qz] * fabs(det);
        double Gp[3][3], S[3][3], cv[3];
        for (int d = 0; d < 3; ++d)
            for (int k = 0; k < 3; ++k)
                Gp[d][k] = G[d][0][q] * Jinv[0][k] + G[d][1][q] * Jinv[1][k] + G[d][2][q] * Jinv[2][k];{lin}
        for (int d = 0; d < 3; ++d)
            for (int k = 0; k < 3; ++k)
                S[d][k] = {float(nu)!r} * Gp[d][k] - (d == k ? P[q] : 0.0);
        for (int d = 0; d < 3; ++d)
            for (int m = 0; m < 3; ++m)
                G[d][m][q] = wd * (Jinv[m][0] * S[d][0] + Jinv[m][1] * S[d][1] + Jinv[m][2] * S[d][2]);
        for (int d = 0; d < 3; ++d) U[d][q] = wd * ({float(beta)!r} * U[d][q] + cv[d]);
        T[q] = -wd * (Gp[0][0] + Gp[1][1] + Gp[2][2]);
    }}
    for (int d = 0; d < 3; ++d) {{
        el_tensor(EB, EB, EB, 1, U[d], c);
        el_tensor(ED, EB, EB, 1, G[d][0], t);  for (int i = 0; i < END; ++i) c[i] += t[i];
        el_tensor(EB, ED, EB, 1, G[d][1], t);  for (int i = 0; i < END; ++i) c[i] += t[i];
        el_tensor(EB, EB, ED, 1, G[d][2], t);  for (int i = 0; i < END; ++i) c[i] += t[i];
        for (int i = 0; i < END; ++i) y[i * 3 + d] += c[i];
    }}
    el_tensor(EQ, EQ, EQ, 1, T, c);
    for (int a = 0; a < ENP; ++a) for (int b = 0; b < ENP; ++b) for (int e = 0; e < ENP; ++e)
        y[3 * END + (a * ENP + b) * ENP + e] += c[(a * EN + b) * EN + e];
}}
#undef ENP
#undef END
#undef EN
"""
    return CStringKernel(code, name)


def assemble_navier_stokes_generic(F: "NavierStokes", up: op2.MixedDat, w: op2.MixedDat = None, tensor=None):
    """The residual R(up) of :class:`NavierStokes` (``w`` None) or the Jacobian action J(up[0]) w through the
    generic wrapper path (:func:`navier_stokes_kernel`): the cross-check and the baseline of the hand-written
    kernels."""
    V = F.V
    if tensor is None:
        tensor = F.dat()
    tensor.zero()
    for d in tensor:
        d.device_ptr
    mm = op2.MixedMap([V.cell_node_map, F.pressure_map])
    k = navier_stokes_kernel(V.degree, F.nu, F.beta, jacobian=w is not None)
    ins = [w(op2.READ, mm), up[0](op2.READ, V.cell_node_map)] if w is not None else [up(op2.READ, mm)]
    op2.par_loop(k, V.cell_set, tensor(op2.INC, mm), V.coordinates(op2.READ, V.coord_map), *ins)
    return tensor


def advection_diffusion_kernel(degree, alpha=1.0, beta=0.0, name="advection_diffusion_action"):
    """C source of the 1-form ``action(alpha*inner(grad(u), grad(v))*dx + inner(dot(b, grad(u)), v)*dx +
    beta*inner(u, v)*dx, u)`` on the scalar Q_p (x) P_p space, with the velocity b of 3 values per node
    (AoS), written the way TSFC's spectral mode would, with J^{-1} formed explicitly, and run through the
    generic wrapper builder: the independent statement of the hand-written FDB_FORM_ADVECTION_DIFFUSION
    kernel.  Arguments: y (INC), coords, u, b.  Degrees 1..3: at degree 4 the NVRTC build of this statement
    reads b at a cell's first node as u there (its host build is exact), so it is refused (DESIGN.md
    section 4.10)."""
    from .codegen import CStringKernel
    if not 1 <= degree <= 3:
        raise NotImplementedError(f"advection_diffusion_kernel: degree {degree} outside 1..3 (the device build of "
                                  f"the degree-4 statement is wrong at a cell's first node, DESIGN.md section 4.10)")
    code = _vector_hex_tables(degree) + f"""static void {name}(double *y, const double *X, const double *u,
                                 const double *b)
{{
    double U[END], G[3][END], Bq[3][END], c[END], t[END];
    for (int d = 0; d < 3; ++d) {{
        for (int i = 0; i < END; ++i) c[i] = b[i * 3 + d];
        el_tensor(EB, EB, EB, 0, c, Bq[d]);
    }}
    el_tensor(EB, EB, EB, 0, u, U);
    el_tensor(ED, EB, EB, 0, u, G[0]);
    el_tensor(EB, ED, EB, 0, u, G[1]);
    el_tensor(EB, EB, ED, 0, u, G[2]);
    for (int qx = 0; qx < EN; ++qx) for (int qy = 0; qy < EN; ++qy) for (int qz = 0; qz < EN; ++qz) {{
        const int q = (qx * EN + qy) * EN + qz;
        const double xi[3] = {{EX[qx], EX[qy], EX[qz]}};
        double J[3][3] = {{{{0}}}};
        for (int v = 0; v < 8; ++v) {{
            const int bv[3] = {{(v >> 2) & 1, (v >> 1) & 1, v & 1}};
            for (int r = 0; r < 3; ++r) {{
                double g = bv[r] ? 1.0 : -1.0;
                for (int e = 0; e < 3; ++e) if (e != r) g *= bv[e] ? xi[e] : 1.0 - xi[e];
                for (int k = 0; k < 3; ++k) J[k][r] += X[v * 3 + k] * g;
            }}
        }}
        /* Jinv[m][k] = dxi_m/dx_k */
        const double det = J[0][0] * (J[1][1] * J[2][2] - J[1][2] * J[2][1])
                         - J[0][1] * (J[1][0] * J[2][2] - J[1][2] * J[2][0])
                         + J[0][2] * (J[1][0] * J[2][1] - J[1][1] * J[2][0]);
        double Jinv[3][3];
        Jinv[0][0] = (J[1][1] * J[2][2] - J[1][2] * J[2][1]) / det;
        Jinv[0][1] = (J[0][2] * J[2][1] - J[0][1] * J[2][2]) / det;
        Jinv[0][2] = (J[0][1] * J[1][2] - J[0][2] * J[1][1]) / det;
        Jinv[1][0] = (J[1][2] * J[2][0] - J[1][0] * J[2][2]) / det;
        Jinv[1][1] = (J[0][0] * J[2][2] - J[0][2] * J[2][0]) / det;
        Jinv[1][2] = (J[0][2] * J[1][0] - J[0][0] * J[1][2]) / det;
        Jinv[2][0] = (J[1][0] * J[2][1] - J[1][1] * J[2][0]) / det;
        Jinv[2][1] = (J[0][1] * J[2][0] - J[0][0] * J[2][1]) / det;
        Jinv[2][2] = (J[0][0] * J[1][1] - J[0][1] * J[1][0]) / det;
        const double wd = EW[qx] * EW[qy] * EW[qz] * fabs(det);
        double gp[3];                                /* grad u */
        for (int k = 0; k < 3; ++k) gp[k] = G[0][q] * Jinv[0][k] + G[1][q] * Jinv[1][k] + G[2][q] * Jinv[2][k];
        for (int m = 0; m < 3; ++m)
            G[m][q] = {float(alpha)!r} * wd * (Jinv[m][0] * gp[0] + Jinv[m][1] * gp[1] + Jinv[m][2] * gp[2]);
        U[q] = wd * ({float(beta)!r} * U[q] + Bq[0][q] * gp[0] + Bq[1][q] * gp[1] + Bq[2][q] * gp[2]);
    }}
    el_tensor(EB, EB, EB, 1, U, c);
    el_tensor(ED, EB, EB, 1, G[0], t);  for (int i = 0; i < END; ++i) c[i] += t[i];
    el_tensor(EB, ED, EB, 1, G[1], t);  for (int i = 0; i < END; ++i) c[i] += t[i];
    el_tensor(EB, EB, ED, 1, G[2], t);  for (int i = 0; i < END; ++i) c[i] += t[i];
    for (int i = 0; i < END; ++i) y[i] += c[i];
}}
#undef END
#undef EN
"""
    return CStringKernel(code, name)


def assemble_advection_diffusion_generic(V: "FunctionSpace", u: op2.Dat, b: op2.Dat, alpha=1.0, beta=0.0,
                                         tensor=None):
    """``assemble(action(a, u))`` of advection-diffusion through the generic wrapper path
    (:func:`advection_diffusion_kernel`): the cross-check and the baseline of :class:`AdvectionDiffusion`."""
    if V.cdim != 1:
        raise ValueError("advection-diffusion takes scalar spaces only")
    if tensor is None:
        tensor = V.dat()
    tensor.zero()
    tensor.device_ptr
    op2.par_loop(advection_diffusion_kernel(V.degree, alpha, beta), V.cell_set, tensor(op2.INC, V.cell_node_map),
                 V.coordinates(op2.READ, V.coord_map), u(op2.READ, V.cell_node_map), b(op2.READ, V.cell_node_map))
    return tensor


def boundary_mass_kernel(degree, gamma=1.0, cdim=1, rank=1, name=None):
    """C source of the exterior-facet form ``gamma*inner(u, v)*ds`` on Q_p (x) P_p hexes with trilinear
    geometry, written the way TSFC would (the whole cell's basis at every facet point, the surface measure
    |dx/dxi_s x dx/dxi_t| of the facet), for the generic wrapper builder: the independent statement of the
    hand-written FDB_FORM_BOUNDARY_MASS kernel.  ``rank`` 1: the action, arguments y (INC), coords, u,
    facet; ``rank`` 2: the element matrix (cdim blocks), arguments A, coords, facet.  ``facet`` is the
    uint32 local facet number 2*direction + side (firedrake_loopy.py:317-381)."""
    from .codegen import CStringKernel
    from .fiat_lite import interval_element
    if cdim not in (1, 3) or rank not in (1, 2):
        raise ValueError("boundary_mass_kernel: cdim 1 or 3, rank 1 or 2")
    el = interval_element(degree)
    n, nd = degree + 1, (degree + 1) ** 3
    Bend, _ = el.tabulate([0.0, 1.0])
    tab = lambda a: "{" + ", ".join("{" + ", ".join(repr(float(v)) for v in r) + "}" for r in a) + "}"
    vec = lambda a: "{" + ", ".join(repr(float(v)) for v in a) + "}"
    name = name or f"boundary_mass{rank}_c{cdim}"
    if rank == 1:
        sig = "double *A, const double *X, const double *u, const unsigned int *facet"
        body = f"""for (int c = 0; c < {cdim}; ++c) {{
            double v = 0.0;
            for (int i = 0; i < {nd}; ++i) v += phi[i] * u[i * {cdim} + c];
            for (int i = 0; i < {nd}; ++i) A[i * {cdim} + c] += wd * phi[i] * v;
        }}"""
    else:
        sig = "double *A, const double *X, const unsigned int *facet"
        body = f"""for (int i = 0; i < {nd}; ++i) for (int j = 0; j < {nd}; ++j)
            for (int c = 0; c < {cdim}; ++c) A[(i * {cdim} + c) * {nd * cdim} + j * {cdim} + c] += wd * phi[i] * phi[j];"""
    code = f"""
static const double MB[{n}][{n}] = {tab(el.B)};      /* basis a at Gauss point q: MB[q][a] */
static const double ME[2][{n}] = {tab(Bend)};        /* basis at the interval's ends */
static const double MX[{n}] = {vec(el.xq)};
static const double MW[{n}] = {vec(el.wq)};
static void {name}({sig})
{{
    const int fd = (int)facet[0] / 2, fs = (int)facet[0] % 2;     /* normal direction, side */
    const int d1 = fd == 0 ? 1 : 0, d2 = fd == 2 ? 1 : 2;           /* tangential directions */
    for (int q1 = 0; q1 < {n}; ++q1) for (int q2 = 0; q2 < {n}; ++q2) {{
        double xi[3], J[3][3], phi[{nd}];
        const double *T[3];
        xi[fd] = (double)fs; xi[d1] = MX[q1]; xi[d2] = MX[q2];
        T[fd] = ME[fs]; T[d1] = MB[q1]; T[d2] = MB[q2];
        for (int c = 0; c < 3; ++c) for (int d = 0; d < 3; ++d) J[c][d] = 0.0;
        for (int v = 0; v < 8; ++v) {{
            const int b[3] = {{(v >> 2) & 1, (v >> 1) & 1, v & 1}};
            for (int d = 0; d < 3; ++d) {{
                double g = b[d] ? 1.0 : -1.0;
                for (int e = 0; e < 3; ++e) if (e != d) g *= b[e] ? xi[e] : 1.0 - xi[e];
                for (int c = 0; c < 3; ++c) J[c][d] += X[v * 3 + c] * g;
            }}
        }}
        const double cx = J[1][d1] * J[2][d2] - J[2][d1] * J[1][d2];
        const double cy = J[2][d1] * J[0][d2] - J[0][d1] * J[2][d2];
        const double cz = J[0][d1] * J[1][d2] - J[1][d1] * J[0][d2];
        const double wd = {float(gamma)!r} * MW[q1] * MW[q2] * sqrt(cx * cx + cy * cy + cz * cz);
        for (int a = 0; a < {n}; ++a) for (int b = 0; b < {n}; ++b) for (int c = 0; c < {n}; ++c)
            phi[(a * {n} + b) * {n} + c] = T[0][a] * T[1][b] * T[2][c];
        {body}
    }}
}}
"""
    return CStringKernel(code, name)


def assemble_boundary_mass_generic(V: "FunctionSpace", u: op2.Dat, gamma=1.0, sub_domain="on_boundary", tensor=None):
    """``assemble(action(gamma*inner(u, v)*ds(sub_domain), u))`` through the generic wrapper path
    (:func:`boundary_mass_kernel`) over the same facet sets as :class:`BoundaryMass`: the cross-check and
    the baseline of the hand-written kernel."""
    from . import codegen
    if tensor is None:
        tensor = V.dat()
    tensor.zero()
    tensor.device_ptr
    k = boundary_mass_kernel(V.degree, gamma, V.cdim)
    for fset, fmap, cmap, facet in _boundary_groups(V, sub_domain):
        codegen.par_loop(k, fset, tensor(op2.INC, fmap), V.coordinates(op2.READ, cmap), u(op2.READ, fmap),
                         facet(op2.READ))
    return tensor


def interior_penalty_kernels(degree, alpha, eta, name=None):
    """C sources of the facet terms of :class:`InteriorPenalty` on DQ_p hexes (Gauss-Legendre nodes, trilinear
    geometry), written the way TSFC would (the whole cell's basis and its physical gradient at every facet point,
    n = J^-T n_ref / |J^-T n_ref| of the '+' cell, the surface measure |det J| |J^-T n_ref|), for the generic wrapper
    builder: the independent statement of the hand-written FDB_FORM_INTERIOR_PENALTY and FDB_FORM_DG_BOUNDARY
    kernels.  Returns {"dS_v": action over the vertical interior facets (args y (INC), coords, u, facets uint[2]),
    "dS_h": the same with the pair (5, 4) baked in, for ON_INTERIOR_FACETS over the cells (args y, coords, u),
    "ds": the Nitsche operator terms alpha*(-dot(grad u, n)*v - u*dot(grad v, n) + (eta/h)*u*v)*ds (args y, coords,
    u, facet uint[1])}."""
    from .codegen import CStringKernel
    from .fiat_lite import interval_element
    el = interval_element(degree, variant="gl")
    n, nd = degree + 1, (degree + 1) ** 3
    Bend, Dend = el.tabulate([0.0, 1.0])
    tab = lambda a: "{" + ", ".join("{" + ", ".join(repr(float(v)) for v in r) + "}" for r in a) + "}"
    vec = lambda a: "{" + ", ".join(repr(float(v)) for v in a) + "}"
    base = name or f"interior_penalty{degree}"
    head = f"""
static const double PB[{n}][{n}] = {tab(el.B)};      /* basis a at Gauss point q */
static const double PD[{n}][{n}] = {tab(el.D)};      /* its derivative */
static const double PE[2][{n}] = {tab(Bend)};        /* basis at the interval's ends */
static const double PF[2][{n}] = {tab(Dend)};        /* derivative at the ends */
static const double PX[{n}] = {vec(el.xq)};
static const double PW[{n}] = {vec(el.wq)};
/* one side of a facet at face point (q1, q2): basis values and physical gradients of the cell's {nd} dofs, the
   inverse Jacobian K (K[d][c] = dxi_d/dx_c) and |det J| */
static double side_tables(const double *X, int f, int q1, int q2, double *phi, double (*grad)[3], double K[3][3])
{{
    const int fd = f / 2, fs = f % 2, d1 = fd == 0 ? 1 : 0, d2 = fd == 2 ? 1 : 2;
    double xi[3], J[3][3];
    const double *T[3], *DT[3];
    xi[fd] = (double)fs; xi[d1] = PX[q1]; xi[d2] = PX[q2];
    T[fd] = PE[fs]; T[d1] = PB[q1]; T[d2] = PB[q2];
    DT[fd] = PF[fs]; DT[d1] = PD[q1]; DT[d2] = PD[q2];
    for (int c = 0; c < 3; ++c) for (int d = 0; d < 3; ++d) J[c][d] = 0.0;
    for (int v = 0; v < 8; ++v) {{
        const int b[3] = {{(v >> 2) & 1, (v >> 1) & 1, v & 1}};
        for (int d = 0; d < 3; ++d) {{
            double g = b[d] ? 1.0 : -1.0;
            for (int e = 0; e < 3; ++e) if (e != d) g *= b[e] ? xi[e] : 1.0 - xi[e];
            for (int c = 0; c < 3; ++c) J[c][d] += X[v * 3 + c] * g;
        }}
    }}
    const double det = J[0][0] * (J[1][1] * J[2][2] - J[1][2] * J[2][1])
                     - J[0][1] * (J[1][0] * J[2][2] - J[1][2] * J[2][0])
                     + J[0][2] * (J[1][0] * J[2][1] - J[1][1] * J[2][0]);
    for (int d = 0; d < 3; ++d) for (int c = 0; c < 3; ++c) {{
        const int d1_ = (d + 1) % 3, d2_ = (d + 2) % 3, c1 = (c + 1) % 3, c2 = (c + 2) % 3;
        K[d][c] = (J[c1][d1_] * J[c2][d2_] - J[c1][d2_] * J[c2][d1_]) / det;   /* cofactor of J[c][d] */
    }}
    for (int a = 0; a < {n}; ++a) for (int b = 0; b < {n}; ++b) for (int c = 0; c < {n}; ++c) {{
        const int i = (a * {n} + b) * {n} + c;
        const double r[3] = {{DT[0][a] * T[1][b] * T[2][c], T[0][a] * DT[1][b] * T[2][c], T[0][a] * T[1][b] * DT[2][c]}};
        phi[i] = T[0][a] * T[1][b] * T[2][c];
        for (int e = 0; e < 3; ++e) grad[i][e] = K[0][e] * r[0] + K[1][e] * r[1] + K[2][e] * r[2];
    }}
    return fabs(det);
}}
static double diameter(const double *X)
{{
    double m = 0.0;
    for (int i = 0; i < 8; ++i) for (int j = i + 1; j < 8; ++j) {{
        double s = 0.0;
        for (int c = 0; c < 3; ++c) s += (X[i * 3 + c] - X[j * 3 + c]) * (X[i * 3 + c] - X[j * 3 + c]);
        if (s > m) m = s;
    }}
    return sqrt(m);
}}
/* the unit normal outward from the cell on facet f and the surface measure |det J| |J^-T n_ref| */
static double normal(int f, double det, double K[3][3], double *nrm)
{{
    const int fd = f / 2;
    const double sg = f % 2 ? 1.0 : -1.0;
    const double l = sqrt(K[fd][0] * K[fd][0] + K[fd][1] * K[fd][1] + K[fd][2] * K[fd][2]);
    for (int c = 0; c < 3; ++c) nrm[c] = sg * K[fd][c] / l;
    return det * l;
}}
"""
    interior = """
{{
    const int fac[2] = {{(int)({fp}), (int)({fm})}};
    const double sig = {eta!r} / (0.5 * (diameter(X) + diameter(X + 24)));
    for (int q1 = 0; q1 < {n}; ++q1) for (int q2 = 0; q2 < {n}; ++q2) {{
        double phi[2][{nd}], grad[2][{nd}][3], K[2][3][3], det[2], u[2] = {{0.0, 0.0}}, gu[2][3] = {{{{0.0}}}}, nrm[3];
        for (int s = 0; s < 2; ++s) {{
            det[s] = side_tables(X + 24 * s, fac[s], q1, q2, phi[s], grad[s], K[s]);
            for (int i = 0; i < {nd}; ++i) {{
                u[s] += phi[s][i] * w[s * {nd} + i];
                for (int c = 0; c < 3; ++c) gu[s][c] += grad[s][i][c] * w[s * {nd} + i];
            }}
        }}
        const double W = PW[q1] * PW[q2] * normal(fac[0], det[0], K[0], nrm);
        const double ju = u[0] - u[1];
        double fu = 0.0;
        for (int c = 0; c < 3; ++c) fu += 0.5 * nrm[c] * (gu[0][c] + gu[1][c]);
        for (int s = 0; s < 2; ++s) {{
            const double sv = s ? -1.0 : 1.0;           /* jump(v, n) = sv v n */
            for (int i = 0; i < {nd}; ++i) {{
                double dn = 0.0;
                for (int c = 0; c < 3; ++c) dn += nrm[c] * grad[s][i][c];
                A[s * {nd} + i] += {alpha!r} * W * (-fu * sv * phi[s][i] - 0.5 * ju * dn + sig * ju * sv * phi[s][i]);
            }}
        }}
    }}
}}
"""
    dS_v = f"static void {base}_dS(double *A, const double *X, const double *w, const unsigned int *facet)" + \
        interior.format(fp="facet[0]", fm="facet[1]", eta=float(eta), n=n, nd=nd, alpha=float(alpha))
    dS_h = f"static void {base}_dSh(double *A, const double *X, const double *w)" + \
        interior.format(fp="5", fm="4", eta=float(eta), n=n, nd=nd, alpha=float(alpha))
    ds = f"""static void {base}_ds(double *A, const double *X, const double *w, const unsigned int *facet)
{{
    const int f = (int)facet[0];
    const double pen = {float(eta)!r} / diameter(X);
    for (int q1 = 0; q1 < {n}; ++q1) for (int q2 = 0; q2 < {n}; ++q2) {{
        double phi[{nd}], grad[{nd}][3], K[3][3], nrm[3], u = 0.0, dnu = 0.0;
        const double det = side_tables(X, f, q1, q2, phi, grad, K);
        const double W = PW[q1] * PW[q2] * normal(f, det, K, nrm);
        for (int i = 0; i < {nd}; ++i) {{
            u += phi[i] * w[i];
            for (int c = 0; c < 3; ++c) dnu += nrm[c] * grad[i][c] * w[i];
        }}
        for (int i = 0; i < {nd}; ++i) {{
            double dn = 0.0;
            for (int c = 0; c < 3; ++c) dn += nrm[c] * grad[i][c];
            A[i] += {float(alpha)!r} * W * (-dnu * phi[i] - u * dn + pen * u * phi[i]);
        }}
    }}
}}
"""
    return {"dS_v": CStringKernel(head + dS_v, f"{base}_dS"), "dS_h": CStringKernel(head + dS_h, f"{base}_dSh"),
            "ds": CStringKernel(head + ds, f"{base}_ds")}


def assemble_interior_penalty_generic(F: "InteriorPenalty", u: op2.Dat, tensor=None):
    """The facet terms of ``assemble(action(a, u))`` for an :class:`InteriorPenalty` form through the generic
    wrapper path (:func:`interior_penalty_kernels`): the vertical interior facets x all layers, the horizontal ones as
    ON_INTERIOR_FACETS over the cells, and the Nitsche terms on F's weak_bcs facets -- the cross-check and the
    baseline of the hand-written facet kernels (the cell term is the Helmholtz kernel's and is not included)."""
    from . import codegen
    V = F.V
    if tensor is None:
        tensor = V.dat()
    tensor.zero()
    tensor.device_ptr
    ks = interior_penalty_kernels(V.degree, F.alpha, F.eta)
    for fset, fmap, cmap, pairs in _dg_interior_groups(V):
        if fset.layers == V.mesh.layers:            # the vertical group
            codegen.par_loop(ks["dS_v"], fset, tensor(op2.INC, fmap), V.coordinates(op2.READ, cmap),
                             u(op2.READ, fmap), pairs(op2.READ))
    if V.mesh.nz > 1:
        codegen.par_loop(ks["dS_h"], V.cell_set, tensor(op2.INC, V.cell_node_map),
                         V.coordinates(op2.READ, V.coord_map), u(op2.READ, V.cell_node_map),
                         iteration_region="ON_INTERIOR_FACETS")
    if F.weak_bcs:
        for fset, fmap, cmap, facet in _boundary_groups(V, F.weak_bcs):
            codegen.par_loop(ks["ds"], fset, tensor(op2.INC, fmap), V.coordinates(op2.READ, cmap), u(op2.READ, fmap),
                             facet(op2.READ))
    return tensor


def dg_transport_kernels(degree, name=None):
    """C sources of the transport terms of :class:`DGTransport` on DQ_p hexes (Gauss-Legendre nodes, trilinear
    geometry, b trilinear from the 8 vertex values), written the way TSFC would (the whole cell's basis and its
    physical gradient at every point, n and the surface measure of the '+' cell), for the generic wrapper builder:
    the independent statement of the hand-written FDB_FORM_DG_TRANSPORT kernels.  Returns {"cell": -u*dot(b, grad
    v)*dx (args y (INC), coords, u, b), "dS_v": the upwind flux over the vertical interior facets (args y, coords, u,
    b, facets uint[2]), "dS_h": the same with the pair (5, 4) baked in, for ON_INTERIOR_FACETS over the cells (args y,
    coords, u, b), "ds": the outflow term max(dot(b, n), 0)*u*v*ds (args y, coords, u, b, facet uint[1])}."""
    from .codegen import CStringKernel
    from .fiat_lite import interval_element
    el = interval_element(degree, variant="gl")
    n, nd = degree + 1, (degree + 1) ** 3
    Bend, Dend = el.tabulate([0.0, 1.0])
    tab = lambda a: "{" + ", ".join("{" + ", ".join(repr(float(v)) for v in r) + "}" for r in a) + "}"
    vec = lambda a: "{" + ", ".join(repr(float(v)) for v in a) + "}"
    base = name or f"dg_transport{degree}"
    head = f"""
static const double TB[{n}][{n}] = {tab(el.B)};      /* basis a at Gauss point q */
static const double TD[{n}][{n}] = {tab(el.D)};      /* its derivative */
static const double TE[2][{n}] = {tab(Bend)};        /* basis at the interval's ends */
static const double TF[2][{n}] = {tab(Dend)};        /* derivative at the ends */
static const double TX[{n}] = {vec(el.xq)};
static const double TW[{n}] = {vec(el.wq)};
/* at reference point xi, with the 1-D tables T, DT of each axis there: the values and physical gradients of the
   cell's {nd} basis functions, the inverse Jacobian K (K[d][c] = dxi_d/dx_c), b (trilinear) and |det J| */
static double tables(const double *X, const double *bv, const double xi[3], const double *T[3], const double *DT[3],
                     double *phi, double (*grad)[3], double K[3][3], double *b)
{{
    double J[3][3];
    for (int c = 0; c < 3; ++c) {{ b[c] = 0.0; for (int d = 0; d < 3; ++d) J[c][d] = 0.0; }}
    for (int v = 0; v < 8; ++v) {{
        const int bb[3] = {{(v >> 2) & 1, (v >> 1) & 1, v & 1}};
        double w = 1.0;
        for (int e = 0; e < 3; ++e) w *= bb[e] ? xi[e] : 1.0 - xi[e];
        for (int c = 0; c < 3; ++c) b[c] += w * bv[v * 3 + c];
        for (int d = 0; d < 3; ++d) {{
            double g = bb[d] ? 1.0 : -1.0;
            for (int e = 0; e < 3; ++e) if (e != d) g *= bb[e] ? xi[e] : 1.0 - xi[e];
            for (int c = 0; c < 3; ++c) J[c][d] += X[v * 3 + c] * g;
        }}
    }}
    const double det = J[0][0] * (J[1][1] * J[2][2] - J[1][2] * J[2][1])
                     - J[0][1] * (J[1][0] * J[2][2] - J[1][2] * J[2][0])
                     + J[0][2] * (J[1][0] * J[2][1] - J[1][1] * J[2][0]);
    for (int d = 0; d < 3; ++d) for (int c = 0; c < 3; ++c) {{
        const int d1_ = (d + 1) % 3, d2_ = (d + 2) % 3, c1 = (c + 1) % 3, c2 = (c + 2) % 3;
        K[d][c] = (J[c1][d1_] * J[c2][d2_] - J[c1][d2_] * J[c2][d1_]) / det;   /* cofactor of J[c][d] */
    }}
    for (int a = 0; a < {n}; ++a) for (int b1 = 0; b1 < {n}; ++b1) for (int c = 0; c < {n}; ++c) {{
        const int i = (a * {n} + b1) * {n} + c;
        const double r[3] = {{DT[0][a] * T[1][b1] * T[2][c], T[0][a] * DT[1][b1] * T[2][c], T[0][a] * T[1][b1] * DT[2][c]}};
        phi[i] = T[0][a] * T[1][b1] * T[2][c];
        for (int e = 0; e < 3; ++e) grad[i][e] = K[0][e] * r[0] + K[1][e] * r[1] + K[2][e] * r[2];
    }}
    return fabs(det);
}}
/* the tables of facet f at face point (q1, q2) */
static double face_tables(const double *X, const double *bv, int f, int q1, int q2, double *phi, double (*grad)[3],
                          double K[3][3], double *b)
{{
    const int fd = f / 2, fs = f % 2, d1 = fd == 0 ? 1 : 0, d2 = fd == 2 ? 1 : 2;
    double xi[3];
    const double *T[3], *DT[3];
    xi[fd] = (double)fs; xi[d1] = TX[q1]; xi[d2] = TX[q2];
    T[fd] = TE[fs]; T[d1] = TB[q1]; T[d2] = TB[q2];
    DT[fd] = TF[fs]; DT[d1] = TD[q1]; DT[d2] = TD[q2];
    return tables(X, bv, xi, T, DT, phi, grad, K, b);
}}
/* the unit normal outward from the cell on facet f and the surface measure |det J| |J^-T n_ref| */
static double normal(int f, double det, double K[3][3], double *nrm)
{{
    const int fd = f / 2;
    const double sg = f % 2 ? 1.0 : -1.0;
    const double l = sqrt(K[fd][0] * K[fd][0] + K[fd][1] * K[fd][1] + K[fd][2] * K[fd][2]);
    for (int c = 0; c < 3; ++c) nrm[c] = sg * K[fd][c] / l;
    return det * l;
}}
"""
    cell = f"""static void {base}_cell(double *A, const double *X, const double *w, const double *bv)
{{
    for (int qx = 0; qx < {n}; ++qx) for (int qy = 0; qy < {n}; ++qy) for (int qz = 0; qz < {n}; ++qz) {{
        double phi[{nd}], grad[{nd}][3], K[3][3], b[3], u = 0.0;
        const double xi[3] = {{TX[qx], TX[qy], TX[qz]}};
        const double *T[3] = {{TB[qx], TB[qy], TB[qz]}}, *DT[3] = {{TD[qx], TD[qy], TD[qz]}};
        const double W = TW[qx] * TW[qy] * TW[qz] * tables(X, bv, xi, T, DT, phi, grad, K, b);
        for (int i = 0; i < {nd}; ++i) u += phi[i] * w[i];
        for (int i = 0; i < {nd}; ++i) A[i] -= W * u * (b[0] * grad[i][0] + b[1] * grad[i][1] + b[2] * grad[i][2]);
    }}
}}
"""
    interior = """
{{
    const int fac[2] = {{(int)({fp}), (int)({fm})}};
    for (int q1 = 0; q1 < {n}; ++q1) for (int q2 = 0; q2 < {n}; ++q2) {{
        double phi[2][{nd}], grad[{nd}][3], K[3][3], b[3], bm[3], nrm[3], u[2] = {{0.0, 0.0}};
        const double det = face_tables(X, bv, fac[0], q1, q2, phi[0], grad, K, b);
        const double W = TW[q1] * TW[q2] * normal(fac[0], det, K, nrm);
        face_tables(X + 24, bv + 24, fac[1], q1, q2, phi[1], grad, K, bm);
        for (int s = 0; s < 2; ++s) for (int i = 0; i < {nd}; ++i) u[s] += phi[s][i] * w[s * {nd} + i];
        const double bn = b[0] * nrm[0] + b[1] * nrm[1] + b[2] * nrm[2];
        const double flux = W * bn * (bn >= 0.0 ? u[0] : u[1]);
        for (int i = 0; i < {nd}; ++i) {{
            A[i] += flux * phi[0][i];
            A[{nd} + i] -= flux * phi[1][i];
        }}
    }}
}}
"""
    dS_v = f"static void {base}_dS(double *A, const double *X, const double *w, const double *bv, " \
           f"const unsigned int *facet)" + interior.format(fp="facet[0]", fm="facet[1]", n=n, nd=nd)
    dS_h = f"static void {base}_dSh(double *A, const double *X, const double *w, const double *bv)" + \
        interior.format(fp="5", fm="4", n=n, nd=nd)
    ds = f"""static void {base}_ds(double *A, const double *X, const double *w, const double *bv,
                                  const unsigned int *facet)
{{
    const int f = (int)facet[0];
    for (int q1 = 0; q1 < {n}; ++q1) for (int q2 = 0; q2 < {n}; ++q2) {{
        double phi[{nd}], grad[{nd}][3], K[3][3], b[3], nrm[3], u = 0.0;
        const double det = face_tables(X, bv, f, q1, q2, phi, grad, K, b);
        const double W = TW[q1] * TW[q2] * normal(f, det, K, nrm);
        const double bn = b[0] * nrm[0] + b[1] * nrm[1] + b[2] * nrm[2];
        for (int i = 0; i < {nd}; ++i) u += phi[i] * w[i];
        for (int i = 0; i < {nd}; ++i) A[i] += W * (bn > 0.0 ? bn : 0.0) * u * phi[i];
    }}
}}
"""
    return {"cell": CStringKernel(head + cell, f"{base}_cell"), "dS_v": CStringKernel(head + dS_v, f"{base}_dS"),
            "dS_h": CStringKernel(head + dS_h, f"{base}_dSh"), "ds": CStringKernel(head + ds, f"{base}_ds")}


def assemble_dg_transport_generic(F: "DGTransport", u: op2.Dat, tensor=None):
    """The transport terms of ``assemble(action(a, u))`` for a :class:`DGTransport` form (cell, upwind dS and outflow
    ds; not the Helmholtz or interior penalty parts) through the generic wrapper path (:func:`dg_transport_kernels`),
    over the same facet sets as the hand-written path: the cross-check and the baseline of FDB_FORM_DG_TRANSPORT."""
    from . import codegen
    V, b = F.V, F.b
    if tensor is None:
        tensor = V.dat()
    tensor.zero()
    tensor.device_ptr
    ks = dg_transport_kernels(V.degree)
    codegen.par_loop(ks["cell"], V.cell_set, tensor(op2.INC, V.cell_node_map), V.coordinates(op2.READ, V.coord_map),
                     u(op2.READ, V.cell_node_map), b(op2.READ, V.coord_map))
    for fset, fmap, cmap, pairs in _dg_interior_groups(V):
        if fset.layers == V.mesh.layers:            # the vertical group
            codegen.par_loop(ks["dS_v"], fset, tensor(op2.INC, fmap), V.coordinates(op2.READ, cmap),
                             u(op2.READ, fmap), b(op2.READ, cmap), pairs(op2.READ))
    if V.mesh.nz > 1:
        codegen.par_loop(ks["dS_h"], V.cell_set, tensor(op2.INC, V.cell_node_map),
                         V.coordinates(op2.READ, V.coord_map), u(op2.READ, V.cell_node_map),
                         b(op2.READ, V.coord_map), iteration_region="ON_INTERIOR_FACETS")
    for fset, fmap, cmap, facet in _boundary_groups(V, "on_boundary"):
        codegen.par_loop(ks["ds"], fset, tensor(op2.INC, fmap), V.coordinates(op2.READ, cmap), u(op2.READ, fmap),
                         b(op2.READ, cmap), facet(op2.READ))
    return tensor


def hyperelasticity_kernel(degree, mu, lmbda, beta=0.0, jacobian=False, name=None):
    """C source of the residual of compressible Neo-Hookean hyperelasticity,
    ``inner(P(F), grad(v))*dx + beta*inner(u, v)*dx`` with ``F = I + grad(u)``, ``J = det(F)`` and
    ``P(F) = mu*(F - F^{-T}) + lmbda*ln(J)*F^{-T}`` (arguments: y (INC), coords, u), or with ``jacobian``
    of its Gateaux derivative's action at u, ``inner(dP[grad(w)], grad(v))*dx + beta*inner(w, v)*dx``
    (arguments: y (INC), coords, w, u).  Written the way TSFC's spectral mode would, with the inverse of F
    formed explicitly, and run through the generic wrapper builder: the independent statement of the
    hand-written FDB_FORM_HYPERELASTICITY[_JACOBIAN] kernels."""
    from .codegen import CStringKernel
    if name is None:
        name = "hyperelasticity_jacobian_action" if jacobian else "hyperelasticity_residual"
    args = "double *y, const double *X, const double *w, const double *u" if jacobian else \
        "double *y, const double *X, const double *u"
    mu, lmbda, beta = repr(float(mu)), repr(float(lmbda)), repr(float(beta))
    # the point stress: P(F) or dP[H] with H the gradient of w
    if jacobian:
        stress = f"""
        double A[3][3], C[3][3], trA = 0.0;
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j)
                A[i][j] = Finv[i][0] * H[0][j] + Finv[i][1] * H[1][j] + Finv[i][2] * H[2][j];
        for (int i = 0; i < 3; ++i) trA += A[i][i];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j)
                C[i][j] = A[i][0] * Finv[0][j] + A[i][1] * Finv[1][j] + A[i][2] * Finv[2][j];
        for (int d = 0; d < 3; ++d)
            for (int k = 0; k < 3; ++k)
                S[d][k] = {mu} * H[d][k] + ({mu} - {lmbda} * lnJ) * C[k][d] + {lmbda} * trA * Finv[k][d];"""
    else:
        stress = f"""
        for (int d = 0; d < 3; ++d)
            for (int k = 0; k < 3; ++k)
                S[d][k] = {mu} * (Fd[d][k] - Finv[k][d]) + {lmbda} * lnJ * Finv[k][d];"""
    wv = "w" if jacobian else "u"
    code = _vector_hex_tables(degree) + f"""static void {name}({args})
{{
    double U[3][END], G[3][3][END], GU[3][3][END], c[END], t[END];
    for (int d = 0; d < 3; ++d) {{
        for (int i = 0; i < END; ++i) c[i] = {wv}[i * 3 + d];
        el_tensor(EB, EB, EB, 0, c, U[d]);
        el_tensor(ED, EB, EB, 0, c, G[d][0]);
        el_tensor(EB, ED, EB, 0, c, G[d][1]);
        el_tensor(EB, EB, ED, 0, c, G[d][2]);
        for (int i = 0; i < END; ++i) c[i] = u[i * 3 + d];
        el_tensor(ED, EB, EB, 0, c, GU[d][0]);
        el_tensor(EB, ED, EB, 0, c, GU[d][1]);
        el_tensor(EB, EB, ED, 0, c, GU[d][2]);
    }}
    for (int qx = 0; qx < EN; ++qx) for (int qy = 0; qy < EN; ++qy) for (int qz = 0; qz < EN; ++qz) {{
        const int q = (qx * EN + qy) * EN + qz;
        const double xi[3] = {{EX[qx], EX[qy], EX[qz]}};
        double J[3][3] = {{{{0}}}};
        for (int v = 0; v < 8; ++v) {{
            const int b[3] = {{(v >> 2) & 1, (v >> 1) & 1, v & 1}};
            for (int r = 0; r < 3; ++r) {{
                double g = b[r] ? 1.0 : -1.0;
                for (int e = 0; e < 3; ++e) if (e != r) g *= b[e] ? xi[e] : 1.0 - xi[e];
                for (int k = 0; k < 3; ++k) J[k][r] += X[v * 3 + k] * g;
            }}
        }}
        const double det = J[0][0] * (J[1][1] * J[2][2] - J[1][2] * J[2][1])
                         - J[0][1] * (J[1][0] * J[2][2] - J[1][2] * J[2][0])
                         + J[0][2] * (J[1][0] * J[2][1] - J[1][1] * J[2][0]);
        double Jinv[3][3];
        Jinv[0][0] = (J[1][1] * J[2][2] - J[1][2] * J[2][1]) / det;
        Jinv[0][1] = (J[0][2] * J[2][1] - J[0][1] * J[2][2]) / det;
        Jinv[0][2] = (J[0][1] * J[1][2] - J[0][2] * J[1][1]) / det;
        Jinv[1][0] = (J[1][2] * J[2][0] - J[1][0] * J[2][2]) / det;
        Jinv[1][1] = (J[0][0] * J[2][2] - J[0][2] * J[2][0]) / det;
        Jinv[1][2] = (J[0][2] * J[1][0] - J[0][0] * J[1][2]) / det;
        Jinv[2][0] = (J[1][0] * J[2][1] - J[1][1] * J[2][0]) / det;
        Jinv[2][1] = (J[0][1] * J[2][0] - J[0][0] * J[2][1]) / det;
        Jinv[2][2] = (J[0][0] * J[1][1] - J[0][1] * J[1][0]) / det;
        const double wd = EW[qx] * EW[qy] * EW[qz] * fabs(det);
        double H[3][3], Fd[3][3], Finv[3][3], S[3][3];
        for (int d = 0; d < 3; ++d)
            for (int k = 0; k < 3; ++k) {{
                H[d][k] = G[d][0][q] * Jinv[0][k] + G[d][1][q] * Jinv[1][k] + G[d][2][q] * Jinv[2][k];
                Fd[d][k] = (d == k ? 1.0 : 0.0)
                         + GU[d][0][q] * Jinv[0][k] + GU[d][1][q] * Jinv[1][k] + GU[d][2][q] * Jinv[2][k];
            }}
        const double dF = Fd[0][0] * (Fd[1][1] * Fd[2][2] - Fd[1][2] * Fd[2][1])
                        - Fd[0][1] * (Fd[1][0] * Fd[2][2] - Fd[1][2] * Fd[2][0])
                        + Fd[0][2] * (Fd[1][0] * Fd[2][1] - Fd[1][1] * Fd[2][0]);
        Finv[0][0] = (Fd[1][1] * Fd[2][2] - Fd[1][2] * Fd[2][1]) / dF;
        Finv[0][1] = (Fd[0][2] * Fd[2][1] - Fd[0][1] * Fd[2][2]) / dF;
        Finv[0][2] = (Fd[0][1] * Fd[1][2] - Fd[0][2] * Fd[1][1]) / dF;
        Finv[1][0] = (Fd[1][2] * Fd[2][0] - Fd[1][0] * Fd[2][2]) / dF;
        Finv[1][1] = (Fd[0][0] * Fd[2][2] - Fd[0][2] * Fd[2][0]) / dF;
        Finv[1][2] = (Fd[0][2] * Fd[1][0] - Fd[0][0] * Fd[1][2]) / dF;
        Finv[2][0] = (Fd[1][0] * Fd[2][1] - Fd[1][1] * Fd[2][0]) / dF;
        Finv[2][1] = (Fd[0][1] * Fd[2][0] - Fd[0][0] * Fd[2][1]) / dF;
        Finv[2][2] = (Fd[0][0] * Fd[1][1] - Fd[0][1] * Fd[1][0]) / dF;
        const double lnJ = log(dF);{stress}
        for (int d = 0; d < 3; ++d) {{
            for (int m = 0; m < 3; ++m)
                G[d][m][q] = wd * (Jinv[m][0] * S[d][0] + Jinv[m][1] * S[d][1] + Jinv[m][2] * S[d][2]);
            U[d][q] *= {beta} * wd;
        }}
    }}
    for (int d = 0; d < 3; ++d) {{
        el_tensor(EB, EB, EB, 1, U[d], c);
        el_tensor(ED, EB, EB, 1, G[d][0], t);  for (int i = 0; i < END; ++i) c[i] += t[i];
        el_tensor(EB, ED, EB, 1, G[d][1], t);  for (int i = 0; i < END; ++i) c[i] += t[i];
        el_tensor(EB, EB, ED, 1, G[d][2], t);  for (int i = 0; i < END; ++i) c[i] += t[i];
        for (int i = 0; i < END; ++i) y[i * 3 + d] += c[i];
    }}
}}
#undef END
#undef EN
"""
    return CStringKernel(code, name)


def assemble_hyperelasticity_generic(V: "FunctionSpace", u: op2.Dat, mu, lmbda, beta=0.0, w: op2.Dat = None,
                                     tensor=None):
    """The residual R(u) of :class:`HyperElasticity` (``w`` None) or the Jacobian action J(u) w through the
    generic wrapper path (:func:`hyperelasticity_kernel`): the cross-check and the baseline of the
    hand-written kernels."""
    if V.cdim != 3:
        raise ValueError("hyperelasticity needs a vector space with 3 components")
    if tensor is None:
        tensor = V.dat()
    tensor.zero()
    tensor.device_ptr
    ins = ([w(op2.READ, V.cell_node_map)] if w is not None else []) + [u(op2.READ, V.cell_node_map)]
    op2.par_loop(hyperelasticity_kernel(V.degree, mu, lmbda, beta, jacobian=w is not None), V.cell_set,
                 tensor(op2.INC, V.cell_node_map), V.coordinates(op2.READ, V.coord_map), *ins)
    return tensor


def assemble_functional(V: "FunctionSpace", f: op2.Dat, measure="dx", integrand="avg"):
    """``assemble(f*dx)`` / ``assemble(f*ds_b)`` / ``ds_t`` / ``ds_v`` / ``ds`` for a scalar
    ``f`` in V: rank-0 parloops with a Global INC argument (firedrake/assemble.py
    ZeroFormAssembler :1170-1194; the reduction of pyop2/parloop.py:411-455), through the
    generic wrapper builder.  Extruded exterior facets follow the reference's split:
    bottom / top = iteration regions ON_BOTTOM / ON_TOP over the cells, vertical = the base
    mesh's exterior facets x all layers (firedrake/assemble.py:1810-1850)."""
    from . import codegen
    _refuse_dq(V, "assemble_functional", "its kernels tabulate the GLL element")
    if V.cdim != 1:
        raise NotImplementedError("functionals of scalar fields only")
    if measure == "ds":
        return sum(assemble_functional(V, f, m) for m in ("ds_b", "ds_t", "ds_v"))
    g = op2.Global(1, 0.0)
    p = V.degree
    if measure == "dx":
        codegen.par_loop(functional_kernel(p, "dx"), V.cell_set, g(op2.INC),
                         V.coordinates(op2.READ, V.coord_map), f(op2.READ, V.cell_node_map))
    elif measure in ("ds_b", "ds_t"):
        k = functional_kernel(p, "ds", facet=4 if measure == "ds_b" else 5)
        codegen.par_loop(k, V.cell_set, g(op2.INC), V.coordinates(op2.READ, V.coord_map),
                         f(op2.READ, V.cell_node_map),
                         iteration_region="ON_BOTTOM" if measure == "ds_b" else "ON_TOP",
                         interior_horizontal=False)
    elif measure == "ds_v":
        if not hasattr(V, "_ext_facets"):
            cells, local = V.mesh.exterior_vertical_facets()
            fset = op2.ExtrudedSet(op2.Set(len(cells)), V.mesh.layers)
            V._ext_facets = (
                fset,
                op2.Map(fset, V.node_set, V.V.arity, V.V.cell_node_map[cells], offset=V.V.offset),
                op2.Map(fset, V.vertex_set, 8, V.mesh.coord_map[cells], offset=V.mesh.coord_offset),
                op2.Dat(op2.DataSet(fset, 1), local, dtype=np.uint32))
        fset, fmap, cmap, local = V._ext_facets
        if fset.total_size:
            codegen.par_loop(functional_kernel(p, "ds"), fset, g(op2.INC), V.coordinates(op2.READ, cmap),
                             f(op2.READ, fmap), local(op2.READ))
    elif measure == "dS_h":
        # horizontal interior facets: ON_INTERIOR_FACETS over the cells, every argument packs the
        # cell below ('+') and the cell above ('-') (pyop2/codegen/builder.py:779-800, 840-844)
        k = functional_kernel(p, "dS", facet=(5, 4), integrand=integrand)
        codegen.par_loop(k, V.cell_set, g(op2.INC), V.coordinates(op2.READ, V.coord_map),
                         f(op2.READ, V.cell_node_map), iteration_region="ON_INTERIOR_FACETS")
    elif measure == "dS_v":
        # vertical interior facets: the base mesh's interior facets x all layers; maps list the
        # nodes of cell '+' then of cell '-' (firedrake/cython/dmcommon.pyx:1636-1677)
        if V.dof_dset.halo is not None:
            raise NotImplementedError("dS_v on a partitioned mesh needs an exec halo of cells")
        if not hasattr(V, "_int_facets"):
            cp, cm, local = V.mesh.interior_vertical_facets()
            fset = op2.ExtrudedSet(op2.Set(len(cp)), V.mesh.layers)
            cat = lambda m: np.concatenate([m[cp], m[cm]], axis=1)
            V._int_facets = (
                fset,
                op2.Map(fset, V.node_set, 2 * V.V.arity, cat(V.V.cell_node_map), offset=np.tile(V.V.offset, 2)),
                op2.Map(fset, V.vertex_set, 16, cat(V.mesh.coord_map), offset=np.tile(V.mesh.coord_offset, 2)),
                op2.Dat(op2.DataSet(fset, 2), local, dtype=np.uint32))
        fset, fmap, cmap, local = V._int_facets
        if fset.total_size:
            codegen.par_loop(functional_kernel(p, "dS", integrand=integrand), fset, g(op2.INC),
                             V.coordinates(op2.READ, cmap), f(op2.READ, fmap), local(op2.READ))
    elif measure == "dS":
        return sum(assemble_functional(V, f, m, integrand) for m in ("dS_h", "dS_v"))
    else:
        raise ValueError(f"unknown measure {measure!r}")
    return float(g.data_ro[0])


class DirichletBC:
    """``DirichletBC(V, g, sub_domain)``: node subset + value
    (firedrake/bcs.py:260-457)."""

    def __init__(self, V: FunctionSpace, g, sub_domain):
        _refuse_dq(V, "DirichletBC", "a DQ space has no boundary nodes; impose the condition weakly with "
                   "InteriorPenalty(..., weak_bcs=sub_domain) and nitsche_load")
        self.V = V
        subs = sub_domain if isinstance(sub_domain, (list, tuple)) else [sub_domain]
        self.sub_domains = tuple(subs)
        nodes = np.unique(np.concatenate([V.boundary_nodes(s) for s in subs])).astype(np.int32)
        self.nodes = nodes
        self.node_set = op2.Subset(V.node_set, nodes)
        self.g = g

    def zero(self, dat):
        dat.zero(self.node_set)

    def set(self, dat, val):
        """dat[nodes] = val[nodes] (val a Dat) or the scalar val."""
        from . import _lib
        L = _lib.lib()
        if not hasattr(self, "_dev_nodes"):
            self._dev_nodes = op2.DeviceArray.from_host(self.nodes)
        if isinstance(val, op2.Dat):
            _lib.check(L.fdb_dat_set_nodes(dat.device_ptr, val.device_ptr, dat.cdim,
                                           self._dev_nodes.ptr, len(self.nodes)))
        else:
            _lib.check(L.fdb_dat_set_nodes_scalar(dat.device_ptr, float(val), dat.cdim,
                                                  self._dev_nodes.ptr, len(self.nodes)))
        dat._device_written()

    def apply(self, dat):
        self.set(dat, self.g)

    def lgmap(self):
        lg = np.arange(self.V.node_count, dtype=np.int32)
        lg[self.nodes] = -1
        return lg


_BOUNDARY_SUB_DOMAINS = (1, 2, 3, 4, "bottom", "top")


def _same_name(a, b):
    return type(a) is type(b) and a == b


def _boundary_sub_domains(sub_domain):
    """The sub-domain names of ``ds(sub_domain)`` in canonical order: those :class:`DirichletBC` takes (1..4 =
    x == 0, x == Lx, y == 0, y == Ly; "bottom", "top"; a tuple of them), or "on_boundary" for all six."""
    if isinstance(sub_domain, str) and sub_domain == "on_boundary":
        return _BOUNDARY_SUB_DOMAINS
    subs = sub_domain if isinstance(sub_domain, (list, tuple)) else (sub_domain,)
    for s in subs:
        if not any(_same_name(s, t) for t in _BOUNDARY_SUB_DOMAINS):
            raise ValueError(f"unknown sub_domain {s!r}: 1..4, 'bottom', 'top' or 'on_boundary'")
    return tuple(t for t in _BOUNDARY_SUB_DOMAINS if any(_same_name(s, t) for s in subs))


def _boundary_groups(V: "FunctionSpace", sub_domain):
    """The exterior facets of ``ds(sub_domain)`` on ``V`` as iteration groups ``(facet set, V map, coordinate
    map, local facet numbers)``, built once per space and sub-domain and cached on the space.  Vertical facets
    (sides 1..4) are the base mesh's exterior facets x all layers, as for ``ds_v``; horizontal ones are the base
    columns with one cell layer and the maps of the bottom cells ("bottom", facet 4) or of the top cells, whose
    rows are the bottom rows shifted by (nz - 1) * offset ("top", facet 5).  Facet dofs are cell dofs, so the
    maps are the owning cells' rows and every matrix entry lies in the cell sparsity."""
    if V.dof_dset.halo is not None or V.cell_set.owner_computes:
        raise NotImplementedError("boundary terms on a partitioned space are not implemented: the exec-halo columns "
                                  "would count their facets twice")
    subs = _boundary_sub_domains(sub_domain)
    cache = V.__dict__.setdefault("_boundary_facets", {})
    if subs in cache:
        return cache[subs]
    mesh, W = V.mesh, V.V
    cmap, off = W.cell_node_map.astype(np.int64), np.asarray(W.offset, dtype=np.int64)
    xmap, xoff = mesh.coord_map.astype(np.int64), np.asarray(mesh.coord_offset, dtype=np.int64)
    groups = []

    def group(layers, rows, xrows, local):
        fset = op2.ExtrudedSet(op2.Set(len(local)), layers)
        groups.append((fset,
                       op2.Map(fset, V.node_set, W.arity, np.ascontiguousarray(rows, dtype=np.int32), offset=W.offset),
                       op2.Map(fset, V.vertex_set, 8, np.ascontiguousarray(xrows, dtype=np.int32),
                               offset=mesh.coord_offset),
                       op2.Dat(op2.DataSet(fset, 1), np.ascontiguousarray(local, dtype=np.uint32), dtype=np.uint32)))

    sides = [s for s in subs if not isinstance(s, str)]
    if sides:
        cells, local = mesh.exterior_vertical_facets()
        keep = np.isin(local, np.array(sides, dtype=np.uint32) - 1)
        if keep.any():
            group(mesh.layers, cmap[cells[keep]], xmap[cells[keep]], local[keep])
    horiz = [(4, 0) if s == "bottom" else (5, mesh.nz - 1) for s in subs if isinstance(s, str)]
    if horiz:
        nb = mesh.num_base_cells
        group(2, np.concatenate([cmap + off[None, :] * shift for _, shift in horiz]),
              np.concatenate([xmap + xoff[None, :] * shift for _, shift in horiz]),
              np.concatenate([np.full(nb, f, dtype=np.uint32) for f, _ in horiz]))
    cache[subs] = groups
    return groups


def _boundary_kernel(V, gamma, rank, diagonal=False):
    if V.cdim not in (1, 3):
        raise NotImplementedError(f"boundary terms take scalar spaces or vector spaces of 3 components, got cdim "
                                  f"{V.cdim}")
    return op2.Kernel("boundary_mass", degree=V.degree, alpha=float(gamma), cdim=V.cdim, rank=rank,
                      diagonal=diagonal, integral="exterior_facet")


def _check_ds(form):
    """Validate a form's ``ds`` terms ((gamma, sub_domain) pairs) and build their facet sets."""
    for term in form.ds:
        if not isinstance(term, (tuple, list)) or len(term) != 2:
            raise ValueError(f"ds holds (gamma, sub_domain) pairs, got {term!r}")
        _boundary_groups(form.V, term[1])


class _BoundaryTerms:
    """The exterior-facet parloops of sum_k gamma_k*inner(u, v)*ds(sub_domain_k) on ``V``: one hand-written
    FDB_FORM_BOUNDARY_MASS loop per term and facet group, added into the same output as the cell loop."""

    def __init__(self, V: "FunctionSpace", ds):
        self.V = V
        self.terms = [(float(g), _boundary_groups(V, s)) for g, s in ds]

    def action_loops(self, tensor: op2.Dat, u: op2.Dat, scatter="atomic"):
        V, loops = self.V, []
        for gamma, groups in self.terms:
            for fset, fmap, cmap, facet in groups:
                gk = op2.GlobalKernel(_boundary_kernel(V, gamma, 1), [fmap, cmap], extruded=True, scatter=scatter)
                loops.append(op2.Parloop(gk, fset, [tensor(op2.INC, fmap), V.coordinates(op2.READ, cmap),
                                                    u(op2.READ, fmap), facet(op2.READ)], location="device"))
        return loops

    def diagonal(self, D: op2.Dat):
        V = self.V
        for gamma, groups in self.terms:
            for fset, fmap, cmap, facet in groups:
                op2.par_loop(_boundary_kernel(V, gamma, 1, diagonal=True), fset, D(op2.INC, fmap),
                             V.coordinates(op2.READ, cmap), facet(op2.READ))

    def matrix(self, tensor: op2.Mat, lg):
        V = self.V
        for gamma, groups in self.terms:
            for fset, fmap, cmap, facet in groups:
                op2.par_loop(_boundary_kernel(V, gamma, 2), fset, tensor(op2.INC, (fmap, fmap), lgmaps=lg),
                             V.coordinates(op2.READ, cmap), facet(op2.READ))


@dataclass
class BoundaryMass:
    """gamma*inner(u, v)*ds(sub_domain) on ``V`` (scalar, or vector with 3 components): a symmetric bilinear form
    that lives on exterior facets only.  ``sub_domain`` takes the names :class:`DirichletBC` takes (1..4,
    "bottom", "top", a tuple of them) and "on_boundary" for the whole boundary.

    Its action gives the boundary loads: ``assemble(BoundaryMass(V, 1.0, 2), u=g)`` is ``inner(g, v)*ds(2)``, a
    Neumann flux for a scalar g, a traction for a vector g, and ``assemble(BoundaryMass(V, h, 2), u=u_inf)`` the
    right-hand side of a Robin condition whose operator term is ``ds=((h, 2),)`` on the volume form.
    ``assemble(F)`` gives an aij Mat (degrees 1..4), ``mat_type="matfree"`` an operator with its diagonal
    (degrees 1..5).  Partitioned spaces are refused."""
    V: FunctionSpace
    gamma: float = 1.0
    sub_domain: object = "on_boundary"
    symmetric = True
    cell_integral = False       # no dx term: only the ds loops run

    def __post_init__(self):
        _refuse_dq(self.V, "BoundaryMass", "its kernel gathers the face nodes of CG_p; the DQ boundary loads are "
                   "nitsche_load and dg_flux_load")
        _check_ds(self)

    @property
    def ds(self):
        return ((self.gamma, self.sub_domain),)

    def coefficient_args(self):
        return []

    def kernel(self, rank, diagonal=False):
        return _boundary_kernel(self.V, self.gamma, rank, diagonal)


def _face_vertices(f):
    """The cell-local vertices (bx*2 + by)*2 + bz of local facet f = 2*direction + side, in (s, t) order (s, t: the
    other two reference axes in increasing order)."""
    d, side = int(f) // 2, int(f) % 2
    out = []
    for sa in (0, 1):
        for sb in (0, 1):
            bx, by, bz = {0: (side, sa, sb), 1: (sa, side, sb), 2: (sa, sb, side)}[d]
            out.append((bx * 2 + by) * 2 + bz)
    return np.array(out)


def _check_facet_orientation(xrows, xoff, pairs):
    """The interior-facet kernel pairs face point (s, t) of '+' with face point (s, t) of '-': the face's vertices,
    read through each side's local facet, must be the same vertices in the same order (in the bottom layer and the
    next, hence in all)."""
    xrows = np.asarray(xrows, dtype=np.int64)
    xoff = np.asarray(xoff, dtype=np.int64)
    for fp, fm in {(int(a), int(b)) for a, b in pairs}:
        sel = (pairs[:, 0] == fp) & (pairs[:, 1] == fm)
        vp, vm = _face_vertices(fp), 8 + _face_vertices(fm)
        for layer in (0, 1):
            if not np.array_equal(xrows[sel][:, vp] + layer * xoff[vp], xrows[sel][:, vm] + layer * xoff[vm]):
                raise ValueError(f"interior facets ({fp}, {fm}): the two cells parametrise the face differently")


def _dg_interior_groups(V: "FunctionSpace"):
    """The interior facets of a DQ space as iteration groups ``(facet set, V map, coordinate map, local facet
    pairs)``, built once and cached on the space.  Vertical facets: the base mesh's interior facets x all layers,
    maps = the '+' cell's row followed by the '-' cell's (arity 2 (p+1)^3, 16 vertices, offsets tiled), pairs (1, 0)
    for x-normal and (3, 2) for y-normal facets.  Horizontal facets: the base columns over nz - 1 facet layers,
    rows [row, row + offset] ('+' the cell below), pair (5, 4)."""
    if "_dg_interior" in V.__dict__:
        return V._dg_interior
    mesh, W = V.mesh, V.V
    cmap, off = W.cell_node_map.astype(np.int64), np.asarray(W.offset, dtype=np.int64)
    xmap, xoff = mesh.coord_map.astype(np.int64), np.asarray(mesh.coord_offset, dtype=np.int64)
    groups = []

    def group(layers, rows, xrows, pairs):
        _check_facet_orientation(xrows, np.tile(xoff, 2), pairs)
        fset = op2.ExtrudedSet(op2.Set(len(pairs)), layers)
        groups.append((fset,
                       op2.Map(fset, V.node_set, 2 * W.arity, np.ascontiguousarray(rows, dtype=np.int32),
                               offset=np.tile(W.offset, 2)),
                       op2.Map(fset, V.vertex_set, 16, np.ascontiguousarray(xrows, dtype=np.int32),
                               offset=np.tile(mesh.coord_offset, 2)),
                       op2.Dat(op2.DataSet(fset, 2), np.ascontiguousarray(pairs, dtype=np.uint32), dtype=np.uint32)))

    cp, cm, local = mesh.interior_vertical_facets()
    if len(cp):
        group(mesh.layers, np.concatenate([cmap[cp], cmap[cm]], axis=1), np.concatenate([xmap[cp], xmap[cm]], axis=1),
              local)
    if mesh.nz > 1:
        nb = mesh.num_base_cells
        group(mesh.nz, np.concatenate([cmap, cmap + off[None, :]], axis=1),
              np.concatenate([xmap, xmap + xoff[None, :]], axis=1), np.tile(np.array([5, 4], dtype=np.uint32), (nb, 1)))
    V._dg_interior = groups
    return groups


def _dq_diagonal_kernel(V, alpha, beta):
    """The cell term's diagonal on a DQ space: the Helmholtz diagonal kernel, degrees 1..3."""
    if V.degree > 3:
        raise NotImplementedError(f"the diagonal of the DQ{V.degree} cell term is not implemented (the Helmholtz "
                                  f"diagonal kernel covers degrees 1..3): getDiagonal and pc_type 'jacobi' need "
                                  f"DQ1..DQ3; use pc_type 'none' on DQ4")
    return op2.Kernel("helmholtz", degree=V.degree, alpha=alpha, beta=beta, diagonal=True, element=V.element)


def _dg_boundary_kernel(V, c_m, c_p, c_s, c_f, diagonal=False):
    return op2.Kernel("dg_boundary", degree=V.degree, alpha=float(c_f), beta=float(c_p), c_m=float(c_m),
                      c_s=float(c_s), diagonal=diagonal, integral="exterior_facet", element=V.element)


def _dg_boundary_loops(V, coefs, sub_domain, tensor, u, scatter="atomic"):
    """The FDB_FORM_DG_BOUNDARY parloops of (c_m, c_p, c_s, c_f) on the exterior facets of ``sub_domain``."""
    loops = []
    for fset, fmap, cmap, facet in _boundary_groups(V, sub_domain):
        gk = op2.GlobalKernel(_dg_boundary_kernel(V, *coefs), [fmap, cmap], extruded=True, scatter=scatter)
        loops.append(op2.Parloop(gk, fset, [tensor(op2.INC, fmap), V.coordinates(op2.READ, cmap), u(op2.READ, fmap),
                                            facet(op2.READ)], location="device"))
    return loops


class _DGFacetTerms:
    """The facet parloops of an :class:`InteriorPenalty` form: FDB_FORM_INTERIOR_PENALTY over every interior facet
    group, FDB_FORM_DG_BOUNDARY with Nitsche's (0, alpha*eta, alpha, alpha) over the weak_bcs facets."""

    def __init__(self, form: "InteriorPenalty"):
        self.form = form
        V = form.V
        self.interior = _dg_interior_groups(V)
        self.nitsche = (0.0, form.alpha * form.eta, form.alpha, form.alpha)

    def _kernel(self, diagonal=False):
        F = self.form
        return op2.Kernel("interior_penalty", degree=F.V.degree, alpha=float(F.alpha), beta=float(F.eta),
                          diagonal=diagonal, integral="interior_facet", element=F.V.element)

    def action_loops(self, tensor: op2.Dat, u: op2.Dat, scatter="atomic"):
        V, loops = self.form.V, []
        for fset, fmap, cmap, pairs in self.interior:
            gk = op2.GlobalKernel(self._kernel(), [fmap, cmap], extruded=True, scatter=scatter)
            loops.append(op2.Parloop(gk, fset, [tensor(op2.INC, fmap), V.coordinates(op2.READ, cmap),
                                                u(op2.READ, fmap), pairs(op2.READ)], location="device"))
        if self.form.weak_bcs:
            loops += _dg_boundary_loops(V, self.nitsche, self.form.weak_bcs, tensor, u, scatter)
        return loops

    def diagonal(self, D: op2.Dat):
        V = self.form.V
        for fset, fmap, cmap, pairs in self.interior:
            op2.par_loop(self._kernel(True), fset, D(op2.INC, fmap), V.coordinates(op2.READ, cmap), pairs(op2.READ))
        if self.form.weak_bcs:
            for fset, fmap, cmap, facet in _boundary_groups(V, self.form.weak_bcs):
                op2.par_loop(_dg_boundary_kernel(V, *self.nitsche, diagonal=True), fset, D(op2.INC, fmap),
                             V.coordinates(op2.READ, cmap), facet(op2.READ))


@dataclass
class InteriorPenalty:
    """The symmetric interior penalty (SIPG) discretisation of -div(alpha grad u) + beta u = f on a scalar DQ_p space
    (``FunctionSpace(mesh, p, family="DQ")``, p = 1..4), with h the cell diameter and n the unit normal:

        a(u, v) = alpha*inner(grad u, grad v)*dx + beta*u*v*dx
                  + alpha*( -inner(avg(grad u), jump(v, n)) - inner(jump(u, n), avg(grad v))
                            + (eta/avg(h))*inner(jump(u, n), jump(v, n)) )*dS
                  + alpha*( -dot(grad u, n)*v - u*dot(grad v, n) + (eta/h)*u*v )*ds(weak_bcs)

    Every integral has p+1 Gauss points per axis.  ``eta`` has no default (the user picks the penalty, as in
    Firedrake's demos); 3*(p+1)**2 keeps the operator positive definite on the meshes of the tests.  ``weak_bcs``:
    the sub-domains (the names :class:`DirichletBC` takes, or "on_boundary") where Dirichlet conditions are imposed
    weakly (Nitsche), ``()`` for natural conditions everywhere; the load of a Dirichlet value g is
    :func:`nitsche_load`, a flux :func:`dg_flux_load`.  ``assemble(F, u=x)`` is the action, ``mat_type="matfree"``
    an operator with ``mult`` and ``getDiagonal`` (no assembled matrix; the diagonal for p = 1..3, which is what the
    cell term's diagonal kernel covers); :func:`solve` runs CG with ``pc_type`` "none" or "jacobi" (p = 1..3).  The cell term runs on the Helmholtz kernels with the DQ element's tables; the facet terms
    on FDB_FORM_INTERIOR_PENALTY and FDB_FORM_DG_BOUNDARY."""
    V: FunctionSpace
    alpha: float = 1.0
    beta: float = 0.0
    eta: float = None
    weak_bcs: object = "on_boundary"
    symmetric = True
    ds = ()

    def __post_init__(self):
        if getattr(self.V, "family", "CG") != "DQ":
            raise ValueError("InteriorPenalty takes a DQ space: FunctionSpace(mesh, p, family='DQ')")
        if self.eta is None:
            raise ValueError("InteriorPenalty needs the penalty eta (no default), e.g. 3*(p+1)**2")
        self.eta = float(self.eta)
        if isinstance(self.weak_bcs, list):
            self.weak_bcs = tuple(self.weak_bcs)
        if self.weak_bcs:
            _boundary_groups(self.V, self.weak_bcs)
        _dg_interior_groups(self.V)

    def coefficient_args(self):
        return []

    def kernel(self, rank, diagonal=False):
        """The cell term alpha*inner(grad u, grad v)*dx + beta*u*v*dx on the DQ element."""
        if diagonal:
            return _dq_diagonal_kernel(self.V, self.alpha, self.beta)
        return Form(self.V, self.alpha, self.beta).kernel(rank)

    def facet_terms(self):
        if "_facet_terms" not in self.__dict__:
            self._facet_terms = _DGFacetTerms(self)
        return self._facet_terms


def _dg_load(V, coefs, sub_domain, g, tensor):
    if tensor is None:
        tensor = V.dat()
    tensor.zero()
    for loop in _dg_boundary_loops(V, coefs, sub_domain, tensor, g):
        loop()
    return tensor


def nitsche_load(F: InteriorPenalty, g: op2.Dat, tensor: op2.Dat = None):
    """The Dirichlet load of ``g`` (a Dat on F.V) on F's weak_bcs, alpha*(-g*dot(grad v, n) + (eta/h)*g*v)*ds, for an
    :class:`InteriorPenalty` form or the diffusion part of a :class:`DGTransport` form."""
    if not F.weak_bcs:
        raise ValueError("the form has no weakly imposed Dirichlet sub-domains (weak_bcs=())")
    return _dg_load(F.V, (0.0, F.alpha * F.eta, F.alpha, 0.0), F.weak_bcs, g, tensor)


def dg_flux_load(V: FunctionSpace, g: op2.Dat, sub_domain="on_boundary", tensor: op2.Dat = None):
    """The flux (Neumann) load g*v*ds(sub_domain) of a Dat ``g`` on a DQ space ``V``."""
    if getattr(V, "family", "CG") != "DQ":
        raise ValueError("dg_flux_load takes a DQ space; on CG spaces the load is assemble(BoundaryMass(V, 1, "
                         "sub_domain), u=g)")
    return _dg_load(V, (1.0, 0.0, 0.0, 0.0), sub_domain, g, tensor)


def _dg_transport_kernel(V, integral, diagonal=False, c_out=1.0, c_in=0.0):
    return op2.Kernel("dg_transport", degree=V.degree, integral=integral, diagonal=diagonal, element=V.element,
                      c_out=float(c_out), c_in=float(c_in))


def _dg_transport_boundary_loops(F, tensor, u, c_out, c_in, scatter="atomic"):
    """The FDB_FORM_DG_TRANSPORT exterior-facet parloops of (c_out, c_in) over every boundary facet of F.V."""
    V, loops = F.V, []
    for fset, fmap, cmap, facet in _boundary_groups(V, "on_boundary"):
        gk = op2.GlobalKernel(_dg_transport_kernel(V, "exterior_facet", False, c_out, c_in), [fmap, cmap],
                              extruded=True, scatter=scatter)
        loops.append(op2.Parloop(gk, fset, [tensor(op2.INC, fmap), V.coordinates(op2.READ, cmap), u(op2.READ, fmap),
                                            F.b(op2.READ, cmap), facet(op2.READ)], location="device"))
    return loops


class _DGTransportTerms:
    """The loops of a :class:`DGTransport` form after its transport cell loop: the Helmholtz cell loop (alpha or
    beta nonzero), :class:`InteriorPenalty`'s own facet loops (alpha > 0), the upwind FDB_FORM_DG_TRANSPORT loops over
    every interior facet group and the outflow loops (c_out, c_in) = (1, 0) over every boundary facet."""

    def __init__(self, form: "DGTransport"):
        self.form = form
        V = form.V
        self.interior = _dg_interior_groups(V)
        self.helmholtz = Form(V, form.alpha, form.beta) if (form.alpha or form.beta) else None
        self.sipg = _DGFacetTerms(form) if form.alpha > 0 else None

    def action_loops(self, tensor: op2.Dat, u: op2.Dat, scatter="atomic"):
        F = self.form
        V, loops = F.V, []
        if self.helmholtz is not None:
            gk = op2.GlobalKernel(self.helmholtz.kernel(1), [V.cell_node_map, V.coord_map], extruded=True,
                                  scatter=scatter)
            loops.append(op2.Parloop(gk, V.cell_set, [tensor(op2.INC, V.cell_node_map),
                                                      V.coordinates(op2.READ, V.coord_map),
                                                      u(op2.READ, V.cell_node_map)], location="device"))
        if self.sipg is not None:
            loops += self.sipg.action_loops(tensor, u, scatter)
        for fset, fmap, cmap, pairs in self.interior:
            gk = op2.GlobalKernel(_dg_transport_kernel(V, "interior_facet"), [fmap, cmap], extruded=True,
                                  scatter=scatter)
            loops.append(op2.Parloop(gk, fset, [tensor(op2.INC, fmap), V.coordinates(op2.READ, cmap),
                                                u(op2.READ, fmap), F.b(op2.READ, cmap), pairs(op2.READ)],
                                     location="device"))
        return loops + _dg_transport_boundary_loops(F, tensor, u, 1.0, 0.0, scatter)

    def diagonal(self, D: op2.Dat):
        F = self.form
        V = F.V
        if self.helmholtz is not None:
            op2.par_loop(_dq_diagonal_kernel(V, F.alpha, F.beta), V.cell_set, D(op2.INC, V.cell_node_map),
                         V.coordinates(op2.READ, V.coord_map))
        if self.sipg is not None:
            self.sipg.diagonal(D)
        for fset, fmap, cmap, pairs in self.interior:
            op2.par_loop(_dg_transport_kernel(V, "interior_facet", True), fset, D(op2.INC, fmap),
                         V.coordinates(op2.READ, cmap), F.b(op2.READ, cmap), pairs(op2.READ))
        for fset, fmap, cmap, facet in _boundary_groups(V, "on_boundary"):
            op2.par_loop(_dg_transport_kernel(V, "exterior_facet", True), fset, D(op2.INC, fmap),
                         V.coordinates(op2.READ, cmap), F.b(op2.READ, cmap), facet(op2.READ))


@dataclass
class DGTransport:
    """Upwind DG transport of a scalar DQ_p field (``FunctionSpace(mesh, p, family="DQ")``, p = 1..4) by a velocity
    ``b`` given at the mesh vertices (a Dat on ``op2.DataSet(V.vertex_set, 3)``, interpolated trilinearly), in the
    conservative form of Firedrake's DG_advection demo, with optional reaction and diffusion:

        a(u, v) = - u*dot(b, grad v)*dx + beta*u*v*dx + alpha*inner(grad u, grad v)*dx
                  + dot(b, n('+'))*u_up*(v('+') - v('-'))*dS       (u_up: u on the side b.n points away from)
                  + max(dot(b, n), 0)*u*v*ds                        (outflow)
                  + [alpha > 0] the dS terms and the ds(weak_bcs) Nitsche terms of InteriorPenalty(V, alpha, 0, eta,
                    weak_bcs)

    Every integral has p+1 Gauss points per axis.  b is single-valued on every face, so the flux is exactly
    conservative: ``1^T A q`` is the outflow flux.  The inflow condition u = g enters through the load
    :func:`inflow_load`; Dirichlet values of the diffusion part through :func:`nitsche_load`.  ``assemble(F, u=x)`` is
    the action, ``mat_type="matfree"`` an operator with ``mult`` and ``getDiagonal`` (no assembled matrix; the
    diagonal for p = 1..4 without alpha and beta, p = 1..3 with them); :func:`solve` runs GMRES with ``pc_type``
    "none" or "jacobi", and :func:`ssprk3` steps ``M dq/dt = load - A q`` in time.  The transport terms run on
    FDB_FORM_DG_TRANSPORT, the rest on the kernels of :class:`InteriorPenalty`."""
    V: FunctionSpace
    b: op2.Dat
    beta: float = 0.0
    alpha: float = 0.0
    eta: float = None
    weak_bcs: object = ()
    symmetric = False
    ds = ()

    def __post_init__(self):
        if getattr(self.V, "family", "CG") != "DQ":
            raise ValueError("DGTransport takes a DQ space: FunctionSpace(mesh, p, family='DQ')")
        ds = getattr(self.b, "dataset", None)
        if ds is None or ds.set is not self.V.vertex_set or self.b.cdim != 3:
            raise ValueError("DGTransport's b has 3 values per mesh vertex: a Dat on op2.DataSet(V.vertex_set, 3)")
        self.alpha, self.beta = float(self.alpha), float(self.beta)
        if self.alpha < 0:
            raise ValueError(f"DGTransport: the diffusivity alpha must be >= 0, got {self.alpha}")
        if self.alpha > 0 and self.eta is None:
            raise ValueError("DGTransport with alpha > 0 needs the interior penalty eta (no default), e.g. 3*(p+1)**2")
        if self.eta is not None:
            self.eta = float(self.eta)
        if isinstance(self.weak_bcs, list):
            self.weak_bcs = tuple(self.weak_bcs)
        if self.weak_bcs and not self.alpha > 0:
            raise ValueError("DGTransport's weak_bcs are the Nitsche terms of the diffusion part and need alpha > 0; "
                             "the inflow condition is inflow_load")
        if self.weak_bcs:
            _boundary_groups(self.V, self.weak_bcs)
        _boundary_groups(self.V, "on_boundary")
        _dg_interior_groups(self.V)

    def coefficient_args(self):
        return [self.b(op2.READ, self.V.coord_map)]

    def kernel(self, rank, diagonal=False):
        """The transport cell term - u*dot(b, grad v)*dx (its diagonal with ``diagonal``)."""
        if rank == 2:
            raise NotImplementedError("DGTransport has no assembled matrix: use the action and mat_type 'matfree'")
        return _dg_transport_kernel(self.V, "cell", diagonal)

    def facet_terms(self):
        if "_facet_terms" not in self.__dict__:
            self._facet_terms = _DGTransportTerms(self)
        return self._facet_terms


def inflow_load(F: DGTransport, g: op2.Dat, tensor: op2.Dat = None):
    """The inflow load -min(dot(b, n), 0)*g*v*ds of a boundary value ``g`` (a Dat on F.V) for a
    :class:`DGTransport` form: the right-hand side that imposes u = g where the flow enters."""
    if not isinstance(F, DGTransport):
        raise TypeError("inflow_load takes a DGTransport form")
    if tensor is None:
        tensor = F.V.dat()
    tensor.zero()
    for loop in _dg_transport_boundary_loops(F, tensor, g, 0.0, -1.0):
        loop()
    return tensor


def ssprk3(F: DGTransport, q: op2.Dat, dt, steps, load: op2.Dat = None):
    """Advance ``M dq/dt = load - A q`` by ``steps`` steps of the three-stage strong-stability-preserving Runge-Kutta
    method of Firedrake's DG_advection demo, in place on the device; A is F's operator, M the mass matrix of F.V and
    ``load`` (e.g. :func:`inflow_load`) is constant in time.  With Gauss-Legendre collocation M is exactly diagonal on
    any hex mesh, and M^-1 is the reciprocal of ``assemble(mass(V), u=1)``.  Stability is the caller's: the scheme is
    explicit and dt must satisfy the CFL condition of the mesh, the degree and b (roughly dt <= h / ((2p + 1) |b|)).
    Returns q."""
    from . import _lib
    from . import mg as _mg
    V = F.V
    lib = _lib.lib()
    n = q._data.size
    minv = assemble(mass(V), u=V.dat(np.ones(V.node_count)))
    op2.par_loop(_mg.reciprocal_kernel(1), V.node_set, minv(op2.RW))
    A = ImplicitMatrixContext(F)
    r, s1, s2 = V.dat(), V.dat(), V.dat()
    dt = float(dt)

    def stage(src, dst):
        """dst = src + dt M^-1 (load - A src)"""
        A.mult(src, r)
        if load is not None:
            _lib.check(lib.fdb_vec_aypx(n, -1.0, load.device_ptr, r.device_ptr))
        else:
            _lib.check(lib.fdb_vec_scale(n, -1.0, r.device_ptr))
        _lib.check(lib.fdb_vec_pointwise_mult(n, r.device_ptr, minv.device_ptr, r.device_ptr))
        r._device_written()
        if dst is not src:
            src.copy(dst)
        dst.axpy(dt, r)

    for _ in range(int(steps)):
        stage(q, s1)                                    # q1 = q + dt L(q)
        stage(s1, s1)
        _lib.check(lib.fdb_vec_scale(n, 0.25, s1.device_ptr))
        s1._device_written()
        s1.axpy(0.75, q)                                # q2 = 3/4 q + 1/4 (q1 + dt L(q1))
        stage(s1, s2)
        _lib.check(lib.fdb_vec_scale(n, 1.0 / 3.0, q.device_ptr))
        q._device_written()
        q.axpy(2.0 / 3.0, s2)                           # q = 1/3 q + 2/3 (q2 + dt L(q2))
    return q


def spectral_helmholtz_kernel(degree, alpha=1.0, beta=0.0, coef=False, name=None):
    """C source of the spectral-element Helmholtz action ``alpha*inner(kappa*grad u, grad v)*dx(GLL) +
    beta*inner(u, v)*dx(GLL)`` on CG_p hexes (p = 1..3), written the way TSFC writes a collocated kernel (the whole
    cell's basis gradient at every GLL point, the full Jacobian there), for the generic wrapper builder: the
    independent statement of FDB_FORM_SPECTRAL_HELMHOLTZ[_COEF].  Arguments: y (INC), coordinates, u[, kappa]."""
    from .codegen import CStringKernel
    from .fiat_lite import interval_element
    if not 1 <= degree <= 3:
        raise NotImplementedError(f"spectral_helmholtz_kernel: degree {degree} (1..3 on the generic path)")
    el = interval_element(degree, quadrature="gll")
    n, nd = degree + 1, (degree + 1) ** 3
    tab = lambda a: "{" + ", ".join("{" + ", ".join(repr(float(v)) for v in r) + "}" for r in a) + "}"
    vec = lambda a: "{" + ", ".join(repr(float(v)) for v in a) + "}"
    base = name or f"spectral_helmholtz{degree}{'_coef' if coef else ''}"
    kap = ", const double *kap" if coef else ""
    src = f"""
static const double TD[{n}][{n}] = {tab(el.D)};      /* d l_a / dx at GLL point q (B is the identity) */
static const double TX[{n}] = {vec(el.xq)};
static const double TW[{n}] = {vec(el.wq)};
static void {base}(double *A, const double *X, const double *w{kap})
{{
    for (int qx = 0; qx < {n}; ++qx) for (int qy = 0; qy < {n}; ++qy) for (int qz = 0; qz < {n}; ++qz) {{
        const int q = (qx * {n} + qy) * {n} + qz;
        const double xi[3] = {{TX[qx], TX[qy], TX[qz]}};
        double J[3][3], K[3][3], grad[{nd}][3], gu[3] = {{0.0, 0.0, 0.0}};
        for (int c = 0; c < 3; ++c) for (int d = 0; d < 3; ++d) J[c][d] = 0.0;
        for (int v = 0; v < 8; ++v) {{
            const int bb[3] = {{(v >> 2) & 1, (v >> 1) & 1, v & 1}};
            for (int d = 0; d < 3; ++d) {{
                double g = bb[d] ? 1.0 : -1.0;
                for (int e = 0; e < 3; ++e) if (e != d) g *= bb[e] ? xi[e] : 1.0 - xi[e];
                for (int c = 0; c < 3; ++c) J[c][d] += X[v * 3 + c] * g;
            }}
        }}
        const double det = J[0][0] * (J[1][1] * J[2][2] - J[1][2] * J[2][1])
                         - J[0][1] * (J[1][0] * J[2][2] - J[1][2] * J[2][0])
                         + J[0][2] * (J[1][0] * J[2][1] - J[1][1] * J[2][0]);
        for (int d = 0; d < 3; ++d) for (int c = 0; c < 3; ++c) {{
            const int d1 = (d + 1) % 3, d2 = (d + 2) % 3, c1 = (c + 1) % 3, c2 = (c + 2) % 3;
            K[d][c] = (J[c1][d1] * J[c2][d2] - J[c1][d2] * J[c2][d1]) / det;
        }}
        for (int a = 0; a < {n}; ++a) for (int b = 0; b < {n}; ++b) for (int c = 0; c < {n}; ++c) {{
            const int i = (a * {n} + b) * {n} + c;
            const double r[3] = {{TD[qx][a] * (b == qy) * (c == qz), (a == qx) * TD[qy][b] * (c == qz),
                                 (a == qx) * (b == qy) * TD[qz][c]}};
            for (int e = 0; e < 3; ++e) {{
                grad[i][e] = K[0][e] * r[0] + K[1][e] * r[1] + K[2][e] * r[2];
                gu[e] += grad[i][e] * w[i];
            }}
        }}
        const double W = TW[qx] * TW[qy] * TW[qz] * fabs(det);
        const double s = {repr(float(alpha))} * W{" * kap[q]" if coef else ""};
        for (int i = 0; i < {nd}; ++i)
            A[i] += s * (gu[0] * grad[i][0] + gu[1] * grad[i][1] + gu[2] * grad[i][2]);
        A[q] += {repr(float(beta))} * W * w[q];
    }}
}}
"""
    return CStringKernel(src, base)


@dataclass
class SpectralForm:
    """The spectral-element (SEM) Helmholtz operator on a scalar CG_p space (p = 1..5), integrated with the GLL rule
    at the nodes themselves (Firedrake's ``dx(scheme=gauss_lobatto_legendre_cube_rule(...))``):

        a(u, v) = alpha*inner(kappa*grad(u), grad(v))*dx(GLL) + beta*inner(u, v)*dx(GLL)

    ``kappa``: a nodal scalar Dat on ``V`` (c**2 of the wave equation), or None for 1.  The mass term is diagonal (mass
    lumping): ``lumped_mass(V)`` is ``SpectralForm(V, 0, 1)``'s diagonal.  ``assemble(F, u=x)`` is the action,
    ``assemble(F, mat_type="matfree")`` an :class:`ImplicitMatrixContext` with ``getDiagonal`` at every degree, and
    :func:`solve` runs CG with ``pc_type`` "none" or "jacobi".  There is no assembled matrix (aij), no geometric or
    p-multigrid, and no ds terms; DQ, vector and partitioned spaces are refused.  Runs on
    FDB_FORM_SPECTRAL_HELMHOLTZ[_COEF] (csrc/sem_hex.cu); :func:`leapfrog` steps the wave equation with it."""
    V: FunctionSpace
    alpha: float = 1.0
    beta: float = 0.0
    kappa: op2.Dat | None = None
    ds: tuple = ()
    symmetric = True

    def __post_init__(self):
        V = self.V
        _refuse_dq(V, "SpectralForm", "it is stated on the GLL nodes of CG spaces")
        if V.cdim != 1:
            raise NotImplementedError("SpectralForm takes scalar spaces only (vector spaces are not implemented)")
        if V.dof_dset.halo is not None:
            raise NotImplementedError("SpectralForm on a partitioned space is not implemented")
        if self.ds:
            raise NotImplementedError("SpectralForm has no ds terms (boundary integrals on the GLL rule are not "
                                      "implemented)")
        if not 1 <= V.degree <= 5:
            raise NotImplementedError(f"SpectralForm: degree {V.degree} outside 1..5")
        self.alpha, self.beta = float(self.alpha), float(self.beta)

    def coefficient_args(self):
        """The parloop arguments that follow the coordinates: kappa, read through the argument map."""
        return [] if self.kappa is None else [self.kappa(op2.READ, self.V.cell_node_map)]

    def kernel(self, rank, diagonal=False):
        if rank == 2:
            raise NotImplementedError("SpectralForm has no assembled matrix (aij): there is no assembled SEM "
                                      "matrix; use the action and mat_type 'matfree'")
        return op2.Kernel("spectral_helmholtz" if self.kappa is None else "spectral_helmholtz_coef",
                          degree=self.V.degree, alpha=self.alpha, beta=self.beta, diagonal=diagonal)


def lumped_mass(V: FunctionSpace, rho: op2.Dat = None, tensor: op2.Dat = None):
    """The GLL (lumped) mass diagonal of ``V``, the diagonal of ``SpectralForm(V, 0, 1)``, times the nodal ``rho`` if
    given: under collocation that is exactly the GLL mass of rho*u*v.  A Dat on V."""
    from . import _lib
    m = ImplicitMatrixContext(SpectralForm(V, 0.0, 1.0)).getDiagonal(tensor if tensor is not None else V.dat())
    if rho is not None:
        _lib.check(_lib.lib().fdb_vec_pointwise_mult(m._data.size, m.device_ptr, rho.device_ptr, m.device_ptr))
        m._device_written()
    return m


def wave_dt_bound(F: SpectralForm, m: op2.Dat, steps=30):
    """A stable leapfrog step for ``M u'' + K u = f`` with the lumped M = diag(``m``) and K the operator of ``F``:
    ``2 / sqrt(1.1 * lambda_max(M^-1 K))``, lambda_max from ``steps`` Jacobi-Lanczos steps
    (:func:`mg.jacobi_lanczos_bounds` with ``invdiag = 1/m``) on the SEM action, from a seeded random start.  The
    factor 1.1 covers the Lanczos estimate's approach from below."""
    from . import mg as _mg
    V = F.V
    minv = V.dat()
    m.copy(minv)
    op2.par_loop(_mg.reciprocal_kernel(1), V.node_set, minv(op2.RW))
    b = V.dat(np.random.default_rng(0).standard_normal(V.node_count))
    _, lmax = _mg.jacobi_lanczos_bounds(ImplicitMatrixContext(F), minv, b, steps=steps)
    return 2.0 / np.sqrt(1.1 * lmax)


def ricker(t, f_peak, t0):
    """The Ricker wavelet (1 - 2 (pi f (t - t0))^2) exp(-(pi f (t - t0))^2) of peak frequency ``f_peak`` centred at
    ``t0`` (the source of Firedrake's full-waveform-inversion demo)."""
    a = (np.pi * f_peak * (np.asarray(t, dtype=float) - t0)) ** 2
    return (1.0 - 2.0 * a) * np.exp(-a)


class PointEvaluator:
    """Evaluation of fields of the CG_p space ``V`` at fixed physical ``points`` (m, 3), and its adjoint, the point
    load (Firedrake's ``PointEvaluator`` / ``VertexOnlyMesh`` interpolation and its adjoint).

    The points are located once, on the host: a uniform bin grid narrows each point to the cells whose vertex
    bounding boxes contain it, and Newton's method on the trilinear map gives its reference coordinates, accepted
    within ``[-tol, 1 + tol]^3`` (``tolerance``, default 1e-8).  A point on a shared face, edge or vertex goes to the
    lowest cell number (row ``c*nz + l`` of ``full_cell_node_list``).  ``missing_points_behaviour``: "error" (a point
    in no cell raises, naming its index) or "ignore" (its value is NaN and it loads nothing).  Each point keeps its
    cell's (p+1)^3 node ids and basis weights on the device: ``evaluate`` is ``fdb_point_eval``, ``adjoint``
    ``fdb_point_load``, both bit-reproducible."""

    def __init__(self, V: FunctionSpace, points, tolerance=None, missing_points_behaviour="error"):
        if missing_points_behaviour not in ("error", "ignore"):
            raise ValueError(f"missing_points_behaviour {missing_points_behaviour!r}: 'error' or 'ignore'")
        _refuse_dq(V, "PointEvaluator")
        if V.cdim != 1:
            raise NotImplementedError("PointEvaluator takes scalar spaces only")
        self.V = V
        self.points = np.ascontiguousarray(np.asarray(points, dtype=float).reshape(-1, 3))
        self.tolerance = 1e-8 if tolerance is None else float(tolerance)
        self.cells, self.xi = locate_points(V, self.points, self.tolerance)
        missing = np.flatnonzero(self.cells < 0)
        if len(missing) and missing_points_behaviour == "error":
            raise ValueError(f"PointEvaluator: point {int(missing[0])} ({self.points[missing[0]]}) is not in the mesh "
                             f"({len(missing)} missing); missing_points_behaviour='ignore' gives NaN there")
        self.idx, self.w = point_weights(V, self.cells, self.xi)
        self.npts, self.nper = len(self.points), (V.degree + 1) ** 3
        self._didx = op2.DeviceArray.from_host(self.idx) if self.npts else None
        self._dw = op2.DeviceArray.from_host(self.w) if self.npts else None

    def _eval_into(self, u: op2.Dat, out_ptr):
        from . import _lib
        _lib.check(_lib.lib().fdb_point_eval(self.npts, self.nper, self._didx.ptr, self._dw.ptr, u.device_ptr,
                                             out_ptr), "fdb_point_eval")

    def _load_into(self, a_ptr, scale, y: op2.Dat):
        from . import _lib
        _lib.check(_lib.lib().fdb_point_load(self.npts, self.nper, self._didx.ptr, self._dw.ptr, a_ptr,
                                             float(scale), y.device_ptr), "fdb_point_load")
        y._device_written()

    def evaluate(self, u: op2.Dat, out=None):
        """The values of ``u`` at the points, (m,) on the host (NaN at missing points)."""
        out = np.empty(self.npts) if out is None else out
        if self.npts:
            buf = op2.DeviceArray(8 * self.npts)
            self._eval_into(u, buf.ptr)
            buf.to_host(out)
        return out

    def adjoint(self, values, tensor: op2.Dat = None):
        """The point load ``sum_k values[k] phi_i(x_k)`` (E^T values), a Dat on V (added into ``tensor`` if given)."""
        tensor = self.V.dat() if tensor is None else tensor
        a = np.ascontiguousarray(np.asarray(values, dtype=float).reshape(self.npts))
        if self.npts:
            da = op2.DeviceArray.from_host(a)
            self._load_into(da.ptr, 1.0, tensor)
        return tensor


def _cell_vertices(V):
    """The vertex coordinates (nc, 8, 3) of every cell, row c*nz + l."""
    mesh = V.mesh
    return mesh.coordinates[mesh.coord_space.full_cell_node_list().astype(np.int64)]


_VERTS = np.array([[(v >> 2) & 1, (v >> 1) & 1, v & 1] for v in range(8)], dtype=float)


def _trilinear(Xc, xi):
    """The trilinear maps of cells Xc (k, 8, 3) at reference points xi (k, 3): x (k, 3) and J (k, 3, 3), J[:, i, d] =
    dx_i/dxi_d."""
    f = np.where(_VERTS[None] > 0, xi[:, None, :], 1.0 - xi[:, None, :])              # (k, 8, 3)
    s = np.where(_VERTS > 0, 1.0, -1.0)
    N = f.prod(axis=2)
    dN = np.stack([s[None, :, d] * np.prod(np.delete(f, d, axis=2), axis=2) for d in range(3)], axis=2)
    return np.einsum("kv,kvi->ki", N, Xc), np.einsum("kvd,kvi->kid", dN, Xc)


def _newton(Xc, x, iters=30):
    """Reference coordinates of physical points x (k, 3) under the trilinear maps of cells Xc (k, 8, 3)."""
    xi = np.full(x.shape, 0.5)
    for _ in range(iters):
        X, J = _trilinear(Xc, xi)
        xi = xi - np.linalg.solve(J, (X - x)[..., None])[..., 0]
        xi = np.clip(xi, -1.0, 2.0)              # keep far-away candidates finite
    return xi


def locate_points(V, points, tol):
    """(cell, xi) of every point: the lowest-numbered cell (row c*nz + l) whose trilinear map takes a reference point
    within [-tol, 1 + tol]^3 to it, found through a uniform bin grid over the cells' vertex bounding boxes; cell -1
    for a point in no cell."""
    Xc = _cell_vertices(V)
    nc, m = len(Xc), len(points)
    lo, hi = Xc.min(axis=1), Xc.max(axis=1)
    pad = tol * (hi - lo).max(axis=1, keepdims=True) + 1e-12 * np.abs(hi).max()
    lo, hi = lo - pad, hi + pad
    g0, g1 = lo.min(axis=0), hi.max(axis=0)
    nb = max(1, int(np.ceil(nc ** (1.0 / 3.0))))
    h = np.maximum((g1 - g0) / nb, 1e-300)
    b_lo = np.clip(((lo - g0) / h).astype(np.int64), 0, nb - 1)
    b_hi = np.clip(((hi - g0) / h).astype(np.int64), 0, nb - 1)
    span = (b_hi - b_lo + 1).max(axis=0)
    keys, owners = [], []
    for di in range(span[0]):
        for dj in range(span[1]):
            for dk in range(span[2]):
                b = b_lo + np.array([di, dj, dk])
                ok = (b <= b_hi).all(axis=1)
                keys.append(((b[ok, 0] * nb + b[ok, 1]) * nb + b[ok, 2]))
                owners.append(np.flatnonzero(ok))
    keys, owners = np.concatenate(keys), np.concatenate(owners)
    order = np.lexsort((owners, keys))                    # by bin, then by cell number
    keys, owners = keys[order], owners[order]
    starts = np.searchsorted(keys, np.arange(nb ** 3 + 1))
    pb = np.floor((points - g0) / h).astype(np.int64)
    inside_grid = ((pb >= 0) & (pb < nb)).all(axis=1)
    pkey = np.where(inside_grid, (np.clip(pb[:, 0], 0, nb - 1) * nb + np.clip(pb[:, 1], 0, nb - 1)) * nb
                    + np.clip(pb[:, 2], 0, nb - 1), 0)
    counts = np.where(inside_grid, starts[pkey + 1] - starts[pkey], 0)
    pid = np.repeat(np.arange(m), counts)
    first = np.repeat(starts[pkey] - np.concatenate([[0], np.cumsum(counts)[:-1]]), counts)
    cand = owners[first + np.arange(len(pid))] if len(pid) else np.zeros(0, dtype=np.int64)
    # the candidates' bounding boxes, then Newton
    box = ((points[pid] >= lo[cand]) & (points[pid] <= hi[cand])).all(axis=1)
    pid, cand = pid[box], cand[box]
    cells, xis = np.full(m, -1, dtype=np.int64), np.zeros((m, 3))
    if len(pid):
        xi = _newton(Xc[cand], points[pid])
        ok = ((xi >= -tol) & (xi <= 1.0 + tol)).all(axis=1)
        pid, cand, xi = pid[ok], cand[ok], xi[ok]
        order = np.lexsort((cand, pid))                   # per point, the lowest cell number first
        pid, cand, xi = pid[order], cand[order], xi[order]
        first = np.ones(len(pid), dtype=bool)
        first[1:] = pid[1:] != pid[:-1]
        cells[pid[first]] = cand[first]
        xis[pid[first]] = np.clip(xi[first], 0.0, 1.0)
    return cells, xis


def point_weights(V, cells, xi):
    """(idx, w), each (m, (p+1)^3): the global nodes of each point's cell and the basis weights phi_j(x_k) there;
    idx -1 and w 0 for a missing point (cell -1)."""
    from .fiat_lite import interval_element
    W, nz = V.V, V.mesh.nz
    el = interval_element(V.degree)
    n, m = V.degree + 1, len(cells)
    found = cells >= 0
    idx = np.full((m, n ** 3), -1, dtype=np.int32)
    w = np.zeros((m, n ** 3))
    if found.any():
        B = [el.tabulate(xi[found, d])[0] for d in range(3)]
        w[found] = np.einsum("ka,kb,kc->kabc", B[0], B[1], B[2]).reshape(-1, n ** 3)
        c = cells[found]
        idx[found] = W.cell_node_map[c // nz].astype(np.int64) + (c % nz)[:, None] * W.offset[None, :].astype(np.int64)
    return np.ascontiguousarray(idx), np.ascontiguousarray(w)


def leapfrog(F: SpectralForm, u: op2.Dat, u_prev: op2.Dat, dt, steps, m: op2.Dat, bcs=(), sources=None,
             receivers=None, scatter="coloured"):
    """Step ``M u'' + K u = sum_k r_k(t) delta(x - x_k)`` with the explicit central difference (leapfrog) scheme

        u^{n+1} = 2 u^n - u^{n-1} - dt^2 M^-1 (K u^n - f^n),     M = diag(m) (the lumped mass, :func:`lumped_mass`)

    on the device, ``steps`` times from ``u`` = u^0 and ``u_prev`` = u^{-1}; K is the operator of ``F``.  ``sources``:
    ``(PointEvaluator, amplitudes)`` with amplitudes (steps, nsrc), r_k(t_n) = amplitudes[n, k], uploaded once.
    ``receivers``: a PointEvaluator sampling u^{n+1} after every step into a device trace.  ``bcs``: rigid walls (u =
    0), held by zeroing M^-1 and u, u_prev on their nodes.  Each step is one SEM action, one ``fdb_point_load`` into its
    output, one ``fdb_vec_leapfrog`` pass and one ``fdb_point_eval``; nothing is copied to the host in the loop.  dt
    is the caller's (:func:`wave_dt_bound`).  ``scatter``: "coloured" (the default: the traces are bitwise repeatable
    from run to run) or "atomic".  Returns the traces (steps, nrec) (None without receivers) and leaves ``u`` and
    ``u_prev`` at u^steps and u^{steps-1}."""
    from . import _lib
    if not isinstance(F, SpectralForm):
        raise TypeError("leapfrog takes a SpectralForm")
    V, L = F.V, _lib.lib()
    steps, dt = int(steps), float(dt)
    n = V.node_count
    minv = V.dat()
    m.copy(minv)
    from . import mg as _mg
    op2.par_loop(_mg.reciprocal_kernel(1), V.node_set, minv(op2.RW))
    for bc in bcs:
        bc.zero(minv)
        bc.zero(u)
        bc.zero(u_prev)
    src_amp = None
    if sources is not None:
        src, amp = sources
        amp = np.ascontiguousarray(np.asarray(amp, dtype=float))
        if amp.shape != (steps, src.npts):
            raise ValueError(f"leapfrog: source amplitudes have shape {amp.shape}, need (steps, nsrc) = "
                             f"{(steps, src.npts)}")
        src_amp = op2.DeviceArray.from_host(amp) if amp.size else None
    nrec = receivers.npts if receivers is not None else 0
    traces = op2.DeviceArray(8 * steps * nrec) if nrec and steps else None
    r = V.dat()
    asm = (OneFormAssembler(F, u, scatter=scatter), OneFormAssembler(F, u_prev, scatter=scatter))
    cur, prev = u, u_prev
    minv_ptr = minv.device_ptr
    for s in range(steps):
        asm[s % 2].assemble(tensor=r)                             # r = K u^n
        if src_amp is not None:
            src._load_into(src_amp.ptr + 8 * s * src.npts, -1.0, r)    # r -= f^n
        _lib.check(L.fdb_vec_leapfrog(n, dt * dt, minv_ptr, r.device_ptr, cur.device_ptr, prev.device_ptr),
                   "fdb_vec_leapfrog")
        prev._device_written()
        cur, prev = prev, cur                                    # u^{n+1} is in the old u^{n-1}'s buffer
        if traces is not None:
            receivers._eval_into(cur, traces.ptr + 8 * s * nrec)
    out = None
    if traces is not None:
        out = traces.to_host(np.empty((steps, nrec)))
    if cur is not u:
        # an odd number of steps: u^steps sits in u_prev's buffer; swap the values back
        tmp = V.dat()
        cur.copy(tmp)
        prev.copy(u_prev)
        tmp.copy(u)
    return out


@dataclass
class Form:
    """alpha*inner(grad(u), grad(v))*dx + beta*inner(u, v)*dx on ``V``.

    With ``kappa`` (a scalar Dat on ``V``): alpha*inner(kappa*grad(u), grad(v))*dx +
    beta*inner(u, v)*dx -- a heterogeneous material, or the Jacobian of a nonlinear diffusion
    problem at the current iterate.  Runs on the hand-written coefficient kernel (scalar spaces).

    ``ds``: boundary terms added to the operator, a tuple of ``(gamma, sub_domain)`` pairs, each
    ``gamma*inner(u, v)*ds(sub_domain)`` (a Robin condition's operator term; see :class:`BoundaryMass`)."""
    V: FunctionSpace
    alpha: float = 1.0
    beta: float = 0.0
    kappa: op2.Dat | None = None
    ds: tuple = ()

    def __post_init__(self):
        if self.ds:
            _refuse_dq(self.V, "Form's ds terms", "DQ boundary terms are InteriorPenalty's weak_bcs")
            _check_ds(self)

    def coefficient_args(self):
        """The parloop arguments that follow the coordinates: kappa, read through the argument map."""
        return [] if self.kappa is None else [self.kappa(op2.READ, self.V.cell_node_map)]

    def kernel(self, rank, diagonal=False):
        if getattr(self.V, "family", "CG") == "DQ":
            if rank == 2:
                raise NotImplementedError("a DQ space has no assembled matrix here: use the action and the "
                                          "matrix-free operator (mat_type='matfree')")
            if self.kappa is not None:
                _refuse_dq(self.V, "Form with kappa")
            return op2.Kernel("helmholtz", degree=self.V.degree, alpha=self.alpha, beta=self.beta, rank=rank,
                              affine=self._affine(rank), element=self.V.element)
        if self.kappa is not None:
            if self.V.cdim != 1:
                raise NotImplementedError("coefficient forms take scalar spaces only")
            return op2.Kernel("helmholtz_coef", degree=self.V.degree, alpha=self.alpha, beta=self.beta,
                              rank=rank, diagonal=diagonal)
        return op2.Kernel("helmholtz", degree=self.V.degree, alpha=self.alpha, beta=self.beta,
                          rank=rank, cdim=self.V.cdim, affine=self._affine(rank))

    def _affine(self, rank):
        import os
        # per-cell metric on meshes whose cells are all parallelepipeds (checked on the device;
        # GPU-validated in round 2, FDB_AFFINE=0 opts out)
        return rank == 1 and os.environ.get("FDB_AFFINE", "1") != "0" and self.V.cells_are_affine()


@dataclass
class NonlinearDiffusion:
    """The residual of nonlinear diffusion on ``V`` (scalar), without its source term:

        F(u; v) = alpha*inner(D(u)*grad(u), grad(v))*dx + beta*inner(u, v)*dx,  D(s) = d0 + d1*s + d2*s**2

    ``assemble(F, u=u)`` is the vector R(u); the problem F(u; v) = inner(f, v)*dx is solved by
    :func:`solve_nonlinear` with ``L = assemble(mass(V), u=f)``.  D(u) is evaluated at each Gauss point
    from the interpolated u, as TSFC evaluates a coefficient expression.  ``ds``: linear boundary terms
    ``gamma*inner(u, v)*ds(sub_domain)`` (e.g. Robin cooling), in the residual and in its Jacobian."""
    V: FunctionSpace
    alpha: float = 1.0
    beta: float = 0.0
    d: tuple = (1.0, 0.0, 0.0)
    ds: tuple = ()
    symmetric = False

    def __post_init__(self):
        _refuse_dq(self.V, "NonlinearDiffusion")
        if self.ds:
            _check_ds(self)

    def coefficient_args(self):
        return []

    def kernel(self, rank, diagonal=False):
        if rank != 1 or diagonal:
            raise ValueError("the residual is a 1-form: its matrix and diagonal are those of F.jacobian(u)")
        if self.V.cdim != 1:
            raise NotImplementedError("nonlinear diffusion takes scalar spaces only")
        return op2.Kernel("nonlinear_diffusion", degree=self.V.degree, alpha=self.alpha, beta=self.beta,
                          d=tuple(self.d))

    def jacobian(self, u0: op2.Dat):
        """The Gateaux derivative at ``u0`` (the exact Newton Jacobian, a bilinear form)."""
        return NonlinearDiffusionJacobian(self.V, self.alpha, self.beta, tuple(self.d), u0, self.ds)

    def diffusivity(self, u: op2.Dat, target: op2.Dat = None):
        """D(u) at the nodes of ``V`` (a pointwise node loop): the coefficient of the SPD operator
        ``Form(V, alpha, beta, kappa=D(u))`` that the multigrid preconditioner of the Newton steps uses."""
        if target is None:
            target = self.V.dat()
        d0, d1, d2 = (repr(float(c)) for c in self.d)
        k = op2.Kernel(f"static void nodal_diffusivity(double *k, const double *u) "
                       f"{{ *k = {d0} + u[0] * ({d1} + {d2} * u[0]); }}", "nodal_diffusivity")
        op2.par_loop(k, self.V.node_set, target(op2.WRITE), u(op2.READ))
        return target


@dataclass
class NonlinearDiffusionJacobian:
    """J(u0)[w; v] = alpha*inner(D(u0)*grad(w) + D'(u0)*w*grad(u0), grad(v))*dx + beta*inner(w, v)*dx:
    a bilinear form (``assemble(J, u=w)``, ``assemble(J)``, ``assemble(J, mat_type="matfree")``) whose
    matrix is NOT symmetric when d1 or d2 is nonzero.  ``u0`` is read through the argument map."""
    V: FunctionSpace
    alpha: float
    beta: float
    d: tuple
    u0: op2.Dat
    ds: tuple = ()
    symmetric = False

    def coefficient_args(self):
        return [self.u0(op2.READ, self.V.cell_node_map)]

    def kernel(self, rank, diagonal=False):
        if self.V.cdim != 1:
            raise NotImplementedError("nonlinear diffusion takes scalar spaces only")
        return op2.Kernel("nonlinear_diffusion_jacobian", degree=self.V.degree, alpha=self.alpha, beta=self.beta,
                          rank=rank, diagonal=diagonal, d=tuple(self.d))


@dataclass
class Elasticity:
    """Linear elasticity on a vector space ``V`` (``cdim = 3``):

        a(u, v) = inner(sigma(u), grad(v))*dx + beta*inner(u, v)*dx,
        sigma(u) = 2*mu*sym(grad(u)) + lmbda*tr(sym(grad(u)))*Identity(3)

    A symmetric bilinear form whose element matrices couple the three components.  It works with
    ``assemble(F, u=w)`` (action, degrees 1..4), ``assemble(F)`` (a blocked aij Mat of block size 3,
    degrees 1..3), ``assemble(F, mat_type="matfree")`` and :func:`solve` with ``pc_type`` "none",
    "jacobi" or "mg" (the coarse operators are ``Elasticity(W, mu, lmbda, beta)`` on the coarser
    levels).  Dirichlet conditions constrain every component of their nodes.  ``ds``: boundary terms
    ``gamma*inner(u, v)*ds(sub_domain)`` added to the operator (elastic supports); a traction load is
    ``assemble(BoundaryMass(V, 1.0, sub_domain), u=t)``."""
    V: FunctionSpace
    mu: float
    lmbda: float
    beta: float = 0.0
    ds: tuple = ()
    symmetric = True

    def __post_init__(self):
        _refuse_dq(self.V, "Elasticity")
        if self.ds:
            _check_ds(self)

    def coefficient_args(self):
        return []

    def kernel(self, rank, diagonal=False):
        if self.V.cdim != 3:
            raise ValueError("elasticity needs a vector space with 3 components")
        return op2.Kernel("elasticity", degree=self.V.degree, mu=self.mu, lmbda=self.lmbda, beta=self.beta,
                          rank=rank, diagonal=diagonal, cdim=3)


@dataclass
class HyperElasticity:
    """The residual of compressible Neo-Hookean hyperelasticity on a vector space ``V`` (``cdim = 3``),
    without its load term:

        F = I + grad(u),  J = det(F),
        psi = mu/2*(tr(F^T F) - 3) - mu*ln(J) + lmbda/2*ln(J)**2,
        R(u; v) = inner(P(F), grad(v))*dx + beta*inner(u, v)*dx,  P = dpsi/dF = mu*(F - F^{-T}) + lmbda*ln(J)*F^{-T}

    ``assemble(F, u=u)`` is the vector R(u) (degrees 1..4); the problem R(u; v) = inner(f, v)*dx is
    solved by :func:`solve_nonlinear`.  At u = 0 its Jacobian is ``Elasticity(V, mu, lmbda, beta)``.  A
    point with J <= 0 (an inverted element) makes ln(J) and the residual NaN, as in Firedrake.  ``ds``: linear
    boundary terms ``gamma*inner(u, v)*ds(sub_domain)``, in the residual and in its Jacobian."""
    V: FunctionSpace
    mu: float
    lmbda: float
    beta: float = 0.0
    ds: tuple = ()
    symmetric = True

    def __post_init__(self):
        _refuse_dq(self.V, "HyperElasticity")
        if self.ds:
            _check_ds(self)

    def coefficient_args(self):
        return []

    def kernel(self, rank, diagonal=False):
        if rank != 1 or diagonal:
            raise ValueError("the residual is a 1-form: its matrix and diagonal are those of F.jacobian(u)")
        if self.V.cdim != 3:
            raise ValueError("hyperelasticity needs a vector space with 3 components")
        return op2.Kernel("hyperelasticity", degree=self.V.degree, mu=self.mu, lmbda=self.lmbda, beta=self.beta,
                          cdim=3)

    def jacobian(self, u0: op2.Dat):
        """The Gateaux derivative at ``u0`` (the exact Newton Jacobian, a symmetric bilinear form)."""
        return HyperElasticityJacobian(self.V, self.mu, self.lmbda, self.beta, u0, self.ds)


@dataclass
class HyperElasticityJacobian:
    """J(u0)[w; v] = inner(dP[grad(w)], grad(v))*dx + beta*inner(w, v)*dx with
    dP[H] = mu*H + (mu - lmbda*ln(J))*F^{-T} H^T F^{-T} + lmbda*tr(F^{-1} H)*F^{-T} at F = I + grad(u0):
    a symmetric bilinear form (``assemble(J, u=w)``, ``assemble(J)`` as a blocked aij Mat,
    ``assemble(J, mat_type="matfree")``).  ``u0`` is read through the argument map."""
    V: FunctionSpace
    mu: float
    lmbda: float
    beta: float
    u0: op2.Dat
    ds: tuple = ()
    symmetric = True

    def coefficient_args(self):
        return [self.u0(op2.READ, self.V.cell_node_map)]

    def kernel(self, rank, diagonal=False):
        if self.V.cdim != 3:
            raise ValueError("hyperelasticity needs a vector space with 3 components")
        return op2.Kernel("hyperelasticity_jacobian", degree=self.V.degree, mu=self.mu, lmbda=self.lmbda,
                          beta=self.beta, rank=rank, diagonal=diagonal, cdim=3)


@dataclass
class AdvectionDiffusion:
    """Advection-diffusion of a scalar on ``V`` (``cdim = 1``):

        a(u, v) = alpha*inner(grad(u), grad(v))*dx + inner(dot(b, grad(u)), v)*dx + beta*inner(u, v)*dx

    with the velocity ``b`` a Dat of 3 values per node of ``V`` (``V.vector_dset(3)``, i.e.
    ``op2.DataSet(V.node_set, 3)``), read through the argument map.  beta = 1/dt gives an implicit
    Euler step of a transported scalar.  The form is NOT symmetric: it works with ``assemble(F, u=w)``
    (action, degrees 1..4), ``assemble(F)`` (aij, degrees 1..3), ``assemble(F, mat_type="matfree")``
    (``multTranspose`` is not implemented) and :func:`solve`, whose default Krylov method for it is GMRES."""
    V: FunctionSpace
    b: op2.Dat
    alpha: float = 1.0
    beta: float = 0.0
    ds: tuple = ()
    symmetric = False

    def __post_init__(self):
        _refuse_dq(self.V, "AdvectionDiffusion")
        if self.b.cdim != 3:
            raise ValueError(f"the velocity b has 3 values per node (V.vector_dset(3)), got {self.b.cdim}")
        if self.ds:
            _check_ds(self)

    def coefficient_args(self):
        return [self.b(op2.READ, self.V.cell_node_map)]

    def kernel(self, rank, diagonal=False):
        if self.V.cdim != 1:
            raise NotImplementedError("advection-diffusion takes scalar spaces only")
        return op2.Kernel("advection_diffusion", degree=self.V.degree, alpha=self.alpha, beta=self.beta,
                          rank=rank, diagonal=diagonal)


@dataclass
class Stokes:
    """Stokes flow on Taylor-Hood hexahedra: velocity in the vector space ``V`` (CG_p, ``cdim = 3``) and
    pressure in the scalar space ``Q`` (CG_{p-1}) on the same mesh, p = 2..4 (Q2-Q1, Q3-Q2, Q4-Q3):

        a((u, p), (v, q)) = mu*inner(grad(u), grad(v))*dx + beta*inner(u, v)*dx - p*div(v)*dx - q*div(u)*dx

    beta = 0 is steady Stokes, beta = 1/dt an implicit Euler step of unsteady Stokes.  The form is symmetric
    and indefinite.  Firedrake's Stokes demo writes ``+ q*div(u)``: that is the same system with the pressure
    rows negated; the symmetric sign here makes the transpose the operator itself.

    Vectors are :class:`op2.MixedDat` (velocity, pressure), e.g. ``F.dat()``.  It works with
    ``assemble(F, u=up)`` (the action, a MixedDat), ``assemble(F, mat_type="matfree")`` and :func:`solve`
    (GMRES, optionally with a diagonal Schur-complement fieldsplit preconditioner).  There is no assembled
    matrix.  Dirichlet conditions are on the velocity space ``V``."""
    V: FunctionSpace
    Q: FunctionSpace
    mu: float = 1.0
    beta: float = 0.0
    ds: tuple = ()
    symmetric = True

    def __post_init__(self):
        _refuse_dq(self.V, "Stokes")
        _refuse_dq(self.Q, "Stokes")
        _refuse_taylor_hood_ds(self.ds, "Stokes")
        self.pressure_map = _taylor_hood_pressure_map(self.V, self.Q, "Stokes")

    def dat(self, u=None, p=None):
        """A (velocity, pressure) vector: ``op2.MixedDat([V.dat(u), Q.dat(p)])``."""
        return op2.MixedDat([self.V.dat(u), self.Q.dat(p)])

    def coefficient_args(self):
        return []

    def kernel(self, rank=1, diagonal=False):
        if rank != 1 or diagonal:
            raise NotImplementedError("Stokes is an action only: there is no assembled matrix or diagonal "
                                      "(use mat_type='matfree')")
        return op2.Kernel("stokes", degree=self.V.degree, mu=self.mu, beta=self.beta)


def _refuse_taylor_hood_ds(ds, what):
    if ds:
        raise NotImplementedError(f"boundary terms on the {what} form are not implemented: a velocity Robin or "
                                  f"slip term needs the fused saddle-point kernel to carry facet integrals")


def _taylor_hood_pressure_map(V, Q, what):
    """Check a Taylor-Hood pair (vector CG_p, scalar CG_{p-1}, p = 2..4, one unpartitioned mesh) and return the
    pressure map on the velocity space's cell set (the parloop iterates over one set)."""
    if V.cdim != 3:
        raise ValueError(f"the {what} velocity space is a vector space with 3 components, got cdim {V.cdim}")
    if Q.cdim != 1:
        raise ValueError(f"the {what} pressure space is scalar, got cdim {Q.cdim}")
    if V.mesh is not Q.mesh:
        raise ValueError(f"the {what} velocity and pressure spaces must be on the same mesh")
    if not 2 <= V.degree <= 4 or Q.degree != V.degree - 1:
        raise ValueError(f"Taylor-Hood Q_p-Q_(p-1) with p = 2..4: got velocity degree {V.degree}, pressure "
                         f"degree {Q.degree}")
    if any(W.dof_dset.halo is not None or W.cell_set.owner_computes for W in (V, Q)):
        raise NotImplementedError(f"{what} on a partitioned mesh is not implemented: the velocity and pressure "
                                  f"node sets need their own halo design")
    return op2.Map(V.cell_set, Q.node_set, Q.V.arity, Q.V.cell_node_map, offset=Q.V.offset)


@dataclass
class NavierStokes:
    """The residual of steady incompressible Navier-Stokes on the Taylor-Hood spaces of :class:`Stokes`
    (velocity ``V``, vector CG_p; pressure ``Q``, CG_{p-1}; p = 2..4), without its source term:

        R((u, p); (v, q)) = nu*inner(grad(u), grad(v))*dx + beta*inner(u, v)*dx + inner(dot(grad(u), u), v)*dx
                            - p*div(v)*dx - q*div(u)*dx

    with the Stokes sign convention, so that R at u = 0 is the Stokes action and the Jacobian at u = 0 is
    ``Stokes(V, Q, mu=nu, beta)``.  nu is the kinematic viscosity (1/Re on the unit cavity).  ``assemble(F,
    u=up)`` is R(up), a MixedDat; ``F.jacobian(up)`` the exact Newton Jacobian; :func:`solve_nonlinear` runs
    Newton with matrix-free GMRES and the fieldsplit preconditioner of :func:`_solve_stokes`.  The (p+1)-point
    Gauss rule integrates the div terms exactly, the convective term not."""
    V: FunctionSpace
    Q: FunctionSpace
    nu: float = 1.0
    beta: float = 0.0
    ds: tuple = ()
    symmetric = False

    def __post_init__(self):
        _refuse_dq(self.V, "NavierStokes")
        _refuse_dq(self.Q, "NavierStokes")
        _refuse_taylor_hood_ds(self.ds, "Navier-Stokes")
        self.pressure_map = _taylor_hood_pressure_map(self.V, self.Q, "Navier-Stokes")

    def dat(self, u=None, p=None):
        """A (velocity, pressure) vector: ``op2.MixedDat([V.dat(u), Q.dat(p)])``."""
        return op2.MixedDat([self.V.dat(u), self.Q.dat(p)])

    def coefficient_args(self):
        return []

    def kernel(self, rank=1, diagonal=False):
        if rank != 1 or diagonal:
            raise ValueError("the residual is a 1-form: its operator is F.jacobian(up), a matrix-free action")
        return op2.Kernel("navier_stokes", degree=self.V.degree, mu=self.nu, beta=self.beta)

    def jacobian(self, up: op2.MixedDat):
        """The Gateaux derivative at the velocity ``up[0]``, read in place (a nonsymmetric bilinear form)."""
        return NavierStokesJacobian(self.V, self.Q, self.nu, self.beta, up[0], self.pressure_map)


@dataclass
class NavierStokesJacobian:
    """J(u0)[(w, r); (v, q)] = nu*inner(grad(w), grad(v))*dx + beta*inner(w, v)*dx + inner(dot(grad(w), u0), v)*dx
    + inner(dot(grad(u0), w), v)*dx - r*div(v)*dx - q*div(w)*dx: a nonsymmetric bilinear form on MixedDats
    (``assemble(J, u=wr)``, ``assemble(J, mat_type="matfree")``; no assembled matrix).  ``u0``, a Dat of the
    velocity space, is read through the velocity map."""
    V: FunctionSpace
    Q: FunctionSpace
    nu: float
    beta: float
    u0: op2.Dat
    pressure_map: op2.Map = None
    symmetric = False

    def __post_init__(self):
        if self.pressure_map is None:
            self.pressure_map = _taylor_hood_pressure_map(self.V, self.Q, "Navier-Stokes")

    def dat(self, u=None, p=None):
        return op2.MixedDat([self.V.dat(u), self.Q.dat(p)])

    def coefficient_args(self):
        return [self.u0(op2.READ, self.V.cell_node_map)]

    def kernel(self, rank=1, diagonal=False):
        if rank != 1 or diagonal:
            raise NotImplementedError("the Navier-Stokes Jacobian is an action only: there is no assembled matrix "
                                      "or diagonal (use mat_type='matfree')")
        return op2.Kernel("navier_stokes_jacobian", degree=self.V.degree, mu=self.nu, beta=self.beta)


_TAYLOR_HOOD_FORMS = (Stokes, NavierStokes, NavierStokesJacobian)


class StokesAssembler:
    """Cached assembler of the action (velocity, pressure) -> (y_u, y_p) on MixedDats of a form on the
    Taylor-Hood pair (:class:`Stokes`, :class:`NavierStokes`, :class:`NavierStokesJacobian`), the counterpart
    of :class:`OneFormAssembler`: the parloop is built once and re-run; the form's coefficients (the Jacobian's
    u) follow the pressure."""

    def __init__(self, form: Stokes, up: op2.MixedDat, bcs=(), scatter="atomic"):
        self.form, self.up, self.bcs = form, up, tuple(bcs)
        V = form.V
        self._gk = op2.GlobalKernel(form.kernel(1), [V.cell_node_map, V.coord_map, form.pressure_map],
                                    extruded=True, scatter=scatter)
        self._loop = None

    def assemble(self, tensor=None):
        F = self.form
        V = F.V
        if tensor is None:
            tensor = F.dat()
        if self._loop is None or self._tensor is not tensor:
            self._tensor = tensor
            u, p = self.up
            yu, yp = tensor
            self._loop = op2.Parloop(self._gk, V.cell_set,
                                     [yu(op2.INC, V.cell_node_map), V.coordinates(op2.READ, V.coord_map),
                                      u(op2.READ, V.cell_node_map), yp(op2.INC, F.pressure_map),
                                      p(op2.READ, F.pressure_map)] + F.coefficient_args(), location="device")
        tensor.zero()
        self._loop()
        for bc in self.bcs:
            bc.zero(tensor[0])
        return tensor


class StokesMatrixContext:
    """Matrix-free operator of a Taylor-Hood form (:class:`Stokes`, :class:`NavierStokesJacobian`) on
    MixedDats: ``mult`` zeroes the velocity-BC entries of x, applies the saddle-point action and writes x back
    on the constrained velocity rows (identity there).  The Stokes operator is symmetric, so ``multTranspose``
    is ``mult``; for a nonsymmetric form it raises."""

    def __init__(self, form: Stokes, bcs=()):
        self.form, self.bcs = form, tuple(bcs)
        self._x = form.dat()
        self._assembler = StokesAssembler(form, self._x, ())

    def mult(self, X: op2.MixedDat, Y: op2.MixedDat):
        from . import _lib
        L = _lib.lib()
        for a, b in zip(self._x, X):
            _lib.check(L.fdb_memcpy_d2d(a.device_ptr, b.device_ptr, b.nbytes))
            a._device_written()
        for bc in self.bcs:
            bc.zero(self._x[0])
        self._assembler.assemble(tensor=Y)
        for bc in self.bcs:
            bc.set(Y[0], X[0])
        return Y

    def multTranspose(self, X: op2.MixedDat, Y: op2.MixedDat):
        if not self.form.symmetric:
            raise NotImplementedError(f"multTranspose: {type(self.form).__name__} is not symmetric, and its "
                                      f"transpose action is not implemented")
        return self.mult(X, Y)


class ConvergenceError(RuntimeError):
    """A nonlinear solve that cannot go on (firedrake.exceptions.ConvergenceError); ``reason`` is the
    SNES converged reason, e.g. "DIVERGED_FNORM_NAN"."""

    def __init__(self, msg, reason):
        super().__init__(msg)
        self.reason = reason


def poisson(V):
    return Form(V, 1.0, 0.0)


def helmholtz(V):
    return Form(V, 1.0, 1.0)


def mass(V):
    return Form(V, 0.0, 1.0)


class OneFormAssembler:
    """Cached assembler of ``action(a, u)`` (firedrake/assemble.py:950-977,
    1073-1096: parloops are built once and re-run)."""

    def __init__(self, form: Form, u: op2.Dat, bcs=(), scatter="atomic"):
        self.form, self.u, self.bcs = form, u, tuple(bcs)
        V = form.V
        # a BoundaryMass form has no cell integral; the ds terms of a form add facet loops after the cell loop
        self._gk = op2.GlobalKernel(form.kernel(1), [V.cell_node_map, V.coord_map], extruded=True,
                                    scatter=scatter) if getattr(form, "cell_integral", True) else None
        ds = getattr(form, "ds", ())
        self._ds = _BoundaryTerms(V, ds) if ds else None
        # an interior penalty form adds its interior- and exterior-facet loops after the cell loop
        self._facets = form.facet_terms() if hasattr(form, "facet_terms") else None
        self._scatter = scatter
        self._loop = None
        self._tensor = None

    def assemble(self, tensor=None):
        V = self.form.V
        if tensor is None:
            tensor = V.dat()
        if self._tensor is not tensor:
            self._tensor = tensor
            if self._gk is not None:
                self._loop = op2.Parloop(self._gk, V.cell_set,
                                         [tensor(op2.INC, V.cell_node_map),
                                          V.coordinates(op2.READ, V.coord_map),
                                          self.u(op2.READ, V.cell_node_map)] + self.form.coefficient_args(),
                                         location="device")
            self._ds_loops = self._ds.action_loops(tensor, self.u, self._scatter) if self._ds else []
            if self._facets is not None:
                self._ds_loops += self._facets.action_loops(tensor, self.u, self._scatter)
        tensor.zero()
        if self._loop is not None:
            self._loop()
        for loop in self._ds_loops:
            loop()
        for bc in self.bcs:
            bc.zero(tensor)
        return tensor


def assemble(form: Form, u=None, tensor=None, bcs=(), mat_type="aij"):
    """``assemble(action(a, u))`` when ``u`` is given (-> Dat), else the
    bilinear form: ``mat_type="aij"`` -> :class:`op2.Mat`, ``"is"`` -> :class:`ISMat` (distributed,
    unassembled), ``"matfree"`` -> :class:`ImplicitMatrixContext`."""
    V = form.V
    bcs = tuple(bcs)
    if isinstance(form, _TAYLOR_HOOD_FORMS):
        if u is not None:
            return StokesAssembler(form, u, bcs).assemble(tensor)
        if isinstance(form, NavierStokes):
            raise ValueError("the Navier-Stokes residual is a 1-form: assemble(F, u=up), or its operator "
                             "assemble(F.jacobian(up), mat_type='matfree')")
        if mat_type != "matfree":
            what = "Stokes" if isinstance(form, Stokes) else "the Navier-Stokes Jacobian"
            raise NotImplementedError(f"mat_type {mat_type!r}: {what} has no assembled matrix, use mat_type "
                                      f"'matfree'")
        return StokesMatrixContext(form, bcs)
    if u is not None:
        return OneFormAssembler(form, u, bcs).assemble(tensor)
    if mat_type == "matfree":
        return ImplicitMatrixContext(form, bcs)
    if isinstance(form, SpectralForm):
        raise NotImplementedError(f"mat_type {mat_type!r}: SpectralForm has no assembled matrix (there is no "
                                  f"assembled SEM matrix); use mat_type 'matfree'")
    if getattr(V, "family", "CG") == "DQ":
        raise NotImplementedError(f"mat_type {mat_type!r}: there is no assembled matrix on a DQ space (the facet "
                                  f"terms couple neighbouring cells outside the cell sparsity); use mat_type "
                                  f"'matfree'")
    if tensor is None:
        dsets = (V.node_set, V.node_set) if V.cdim == 1 else (V.dof_dset, V.dof_dset)
        tensor = op2.Mat(op2.Sparsity(dsets, [(V.cell_node_map, V.cell_node_map, None)]))
    tensor.zero()
    lg = None
    if bcs and V.cdim == 1:
        lgm = np.arange(V.node_count, dtype=np.int32)
        for bc in bcs:
            lgm[bc.nodes] = -1
        lg = (lgm, lgm)
    elif bcs:
        # vector-valued space: dof-level lgmap, every component of a constrained node masked
        lgm = np.arange(V.node_count * V.cdim, dtype=np.int32).reshape(-1, V.cdim)
        for bc in bcs:
            lgm[bc.nodes, :] = -1
        lgm = np.ascontiguousarray(lgm.ravel())
        lg = (lgm, lgm)
    if getattr(form, "cell_integral", True):
        op2.par_loop(form.kernel(2), V.cell_set,
                     tensor(op2.INC, (V.cell_node_map, V.cell_node_map), lgmaps=lg),
                     V.coordinates(op2.READ, V.coord_map), *form.coefficient_args())
    if getattr(form, "ds", ()):
        # facet dofs are cell dofs: the facet element matrices go into the same Mat and pattern
        _BoundaryTerms(V, form.ds).matrix(tensor, lg)
    owned = V.node_set.size
    for bc in bcs:
        # on a partitioned space a constrained node gets its unit diagonal from its OWNER only:
        # the ghost copies' rows stay empty and add nothing in the local->global sum of ISMat.mult
        rows = bc.nodes[bc.nodes < owned] if mat_type == "is" else bc.nodes
        tensor.set_local_diagonal_entries(rows, 1.0)
    tensor.assemble()
    if mat_type == "is":
        return ISMat(V, tensor)
    if V.dof_dset.halo is not None:
        raise NotImplementedError("assembled matrices on a partitioned space are mat_type='is' "
                                  "(unassembled, one block per GPU) or 'matfree'")
    return tensor


class ISMat:
    """``mat_type="is"``: the distributed matrix kept UNASSEMBLED, A = sum_r R_r^T A_r R_r with A_r the
    matrix of rank r's owned cells over its owned + ghost dofs (PETSc MATIS, which the reference supports:
    firedrake/assemble.py:1330-1345, pyop2/types/mat.py:930-933).  No matrix entries ever cross GPUs (the
    reference's MatAssembly stash exchange, SURVEY.md section 2.3 C4, disappears); ``mult`` is a local
    SpMV followed by the local->global halo sum that vectors use anyway."""

    def __init__(self, V: FunctionSpace, local: op2.Mat):
        self.V, self.local = V, local

    def mult(self, X: op2.Dat, Y: op2.Dat):
        halo = self.V.dof_dset.halo
        if halo is not None and not X.halo_valid:
            halo.global_to_local_begin(X)
            halo.global_to_local_end(X)
        self.local.mult(X, Y)
        if halo is not None:
            halo.local_to_global_begin(Y)
            halo.local_to_global_end(Y)
        return Y


class ImplicitMatrixContext:
    """Matrix-free operator (firedrake/matrix_free/operators.py:74-242): ``mult``
    = zero the column-BC entries of x, assemble ``action(a, x)``, write x back on
    the row-BC entries (identity on constrained rows).  x and y stay on the
    device across calls (SURVEY.md section 8f row f1)."""

    def __init__(self, form: Form, bcs=()):
        self.form, self.bcs = form, tuple(bcs)
        V = form.V
        self._x = V.dat()
        self._assembler = OneFormAssembler(form, self._x, ())

    def getDiagonal(self, D: op2.Dat):
        """``assemble(a, diagonal=True)`` then 1 on the constrained rows
        (matrix_free/operators.py:199-205; firedrake/assemble.py:1226-1241)."""
        V = self.form.V
        if not getattr(self.form, "cell_integral", True):
            k = None                        # BoundaryMass: the ds loops only
        elif self.form.coefficient_args() or not isinstance(self.form, Form):
            # coefficient forms (kappa, a Jacobian's linearisation point) and elasticity have their own
            # diagonal kernel
            k = self.form.kernel(1, diagonal=True)
        else:
            k = _dq_diagonal_kernel(V, self.form.alpha, self.form.beta) if getattr(V, "element", None) is not None else \
                op2.Kernel("helmholtz", degree=V.degree, alpha=self.form.alpha, beta=self.form.beta, diagonal=True)
        D.zero()
        if k is not None:
            op2.par_loop(k, V.cell_set, D(op2.INC, V.cell_node_map), V.coordinates(op2.READ, V.coord_map),
                         *self.form.coefficient_args())
        if getattr(self.form, "ds", ()):
            _BoundaryTerms(V, self.form.ds).diagonal(D)
        if hasattr(self.form, "facet_terms"):
            self.form.facet_terms().diagonal(D)
        for bc in self.bcs:
            bc.set(D, 1.0)
        return D

    def duplicate(self, copy=True):
        """``MatDuplicate`` of the python-context matrix (matrix_free/operators.py:451-470): a new
        context on the same form and conditions (nothing is assembled, so nothing is copied)."""
        if not copy:
            raise NotImplementedError("cannot duplicate a matrix-free operator without its values (copy=0)")
        return ImplicitMatrixContext(self.form, self.bcs)

    def createSubMatrix(self, row_is, col_is=None):
        """``MatCreateSubMatrix`` (matrix_free/operators.py:380-447).  The spaces here have ONE field,
        so an index set is either the whole dof range -- the reference then rebuilds the context on the
        extracted sub-form, i.e. on the same form -- or an arbitrary one, for which the reference falls
        back to PETSc's virtual sub-matrix (``MatCreateSubMatrixVirtual``: scatter the sub-vector into
        a zero full vector, apply, gather the rows): :class:`SubMatrixContext`."""
        col_is = row_is if col_is is None else col_is
        n = self.form.V.node_count * self.form.V.cdim
        whole = lambda s: len(s) == n and np.array_equal(np.asarray(s), np.arange(n))
        if whole(row_is) and whole(col_is):
            return self.duplicate()
        return SubMatrixContext(self, row_is, col_is)

    def multTranspose(self, X: op2.Dat, Y: op2.Dat):
        """``Y = A^T X`` (matrix_free/operators.py:245-330: the action of ``adjoint(a)`` with the
        row and column conditions exchanged).  Every form of the supported family is
        symmetric and row/column DirichletBCs coincide here (no EquationBC), so A^T = A.  The
        Jacobian of nonlinear diffusion and advection-diffusion are not symmetric, and their transpose
        is not implemented."""
        if not getattr(self.form, "symmetric", True):
            which = "advection-diffusion" if isinstance(self.form, AdvectionDiffusion) else \
                "DG transport" if isinstance(self.form, DGTransport) else "the nonlinear diffusion Jacobian"
            raise NotImplementedError(f"multTranspose of a nonsymmetric form ({which})")
        return self.mult(X, Y)

    def mult(self, X: op2.Dat, Y: op2.Dat):
        from . import _lib
        L = _lib.lib()
        _lib.check(L.fdb_memcpy_d2d(self._x.device_ptr, X.device_ptr, X.nbytes))
        self._x._device_written()
        self._x.halo_valid = False
        for bc in self.bcs:
            bc.zero(self._x)
        self._assembler.assemble(tensor=Y)
        for bc in self.bcs:
            bc.set(Y, X)
        return Y


class SubMatrixContext:
    """Virtual sub-matrix ``A[rows, cols]`` of a matrix-free operator: ``mult(xs, ys)`` with compact
    sub-vectors (plain device Dats of len(cols) / len(rows) entries; dof indices = node*cdim + comp)."""

    def __init__(self, parent, rows, cols):
        self.parent = parent
        self.rows = np.ascontiguousarray(rows, dtype=np.int32)
        self.cols = np.ascontiguousarray(cols, dtype=np.int32)
        self._drows = op2.DeviceArray.from_host(self.rows)
        self._dcols = op2.DeviceArray.from_host(self.cols)
        V = parent.form.V
        self._x, self._y = V.dat(), V.dat()
        self.row_set, self.col_set = op2.Set(len(self.rows)), op2.Set(len(self.cols))

    def mult(self, xs: op2.Dat, ys: op2.Dat):
        from . import _lib
        L = _lib.lib()
        self._x.zero()
        _lib.check(L.fdb_vec_scatter(len(self.cols), self._dcols.ptr, xs.device_ptr, self._x.device_ptr))
        self._x._device_written()
        self.parent.mult(self._x, self._y)
        _lib.check(L.fdb_vec_gather(len(self.rows), self._drows.ptr, self._y.device_ptr, ys.device_ptr))
        ys._device_written()
        return ys


def cg(A, b: op2.Dat, x: op2.Dat, rtol=1e-8, atol=0.0, maxit=1000, allreduce=None):
    """Unpreconditioned conjugate gradients on device-resident Dats (the solve
    of demos/matrix_free/poisson.py.rst:38-47 with ``ksp_type cg, pc_type
    none``).  ``A`` needs ``mult(X, Y)``.  Returns (iterations, residual norms).
    ``allreduce``: callable summing a scalar over ranks (owned dofs only)."""
    V = b.dataset
    r = op2.Dat(V)
    p = op2.Dat(V)
    Ap = op2.Dat(V)
    n_owned = b.dataset.set.size * b.cdim

    def dot(a, c):
        import ctypes as C
        from . import _lib
        out = C.c_double()
        _lib.check(_lib.lib().fdb_vec_dot(n_owned, a.device_ptr, c.device_ptr, C.byref(out)))
        return allreduce(out.value) if allreduce else out.value

    from . import _lib
    L = _lib.lib()
    n = b._data.size
    A.mult(x, Ap)
    _lib.check(L.fdb_memcpy_d2d(r.device_ptr, b.device_ptr, b.nbytes))
    r._device_written()
    _lib.check(L.fdb_vec_axpy(n, -1.0, Ap.device_ptr, r.device_ptr))
    r._device_written()
    _lib.check(L.fdb_memcpy_d2d(p.device_ptr, r.device_ptr, r.nbytes))
    p._device_written()
    rr = dot(r, r)
    r0 = np.sqrt(rr)
    hist = [r0]
    it = 0
    while it < maxit and np.sqrt(rr) > max(rtol * r0, atol):
        A.mult(p, Ap)
        alpha = rr / dot(p, Ap)
        # raw vector updates over all local rows: Ap's ghost rows hold partial sums, so the
        # ghost rows of x, r and p are NOT current afterwards (_device_written invalidates them;
        # A.mult refreshes p's through global_to_local when the operator reads ghosts)
        _lib.check(L.fdb_vec_axpy(n, alpha, p.device_ptr, x.device_ptr))
        x._device_written()
        _lib.check(L.fdb_vec_axpy(n, -alpha, Ap.device_ptr, r.device_ptr))
        r._device_written()
        rr_new = dot(r, r)
        _lib.check(L.fdb_vec_aypx(n, rr_new / rr, r.device_ptr, p.device_ptr))   # p = r + beta p
        p._device_written()
        rr = rr_new
        hist.append(np.sqrt(rr))
        it += 1
    x._device_written()
    return it, hist


def gmres(A, b: op2.Dat, x: op2.Dat, M=None, rtol=1e-5, atol=0.0, restart=30, maxit=10000, allreduce=None):
    """Restarted, right-preconditioned GMRES in its flexible form (``ksp_type fgmres``; with a fixed
    preconditioner it is ``ksp_type gmres`` with right preconditioning) on device-resident Dats.
    The preconditioned vectors z_j = M(v_j) are kept, so ``M`` may change from one application to
    the next, as a V-cycle with an inner Krylov coarse solve does.  ``A`` needs ``mult(X, Y)``; ``M(r,
    z)`` writes z from z = 0 (None: no preconditioner).  Inner products run over the owned dofs,
    summed over the ranks by ``allreduce``; the (restart + 1) x restart Hessenberg least-squares
    problem is solved on the host with Givens rotations.  Converged when the residual norm is at most
    max(rtol * ||b - A x0||, atol).  Returns (iterations, residual norms).

    The vectors may be :class:`op2.MixedDat` (e.g. velocity and pressure of :class:`Stokes`): every vector
    operation then runs block by block, and an inner product is the sum of the blocks' inner products."""
    import ctypes as C
    from . import _lib
    from .mg import _touched
    L = _lib.lib()
    mixed = isinstance(b, op2.MixedDat)
    blocks = (lambda v: tuple(v)) if mixed else (lambda v: (v,))
    sizes = [(d._data.size, d.dataset.set.size * d.cdim) for d in blocks(b)]
    m = max(1, int(restart))
    new = (lambda: op2.MixedDat([op2.Dat(d.dataset) for d in b])) if mixed else (lambda: op2.Dat(b.dataset))
    Vs = [new() for _ in range(m + 1)]
    Zs = [new() for _ in range(m)] if M is not None else Vs
    w = new()

    def dot(u, v):
        s = 0.0
        for (_, n_owned), ub, vb in zip(sizes, blocks(u), blocks(v)):
            out = C.c_double()
            _lib.check(L.fdb_vec_dot(n_owned, ub.device_ptr, vb.device_ptr, C.byref(out)))
            s += out.value
        return allreduce(s) if allreduce else s

    def axpy(a, xv, yv):
        for (n, _), xb, yb in zip(sizes, blocks(xv), blocks(yv)):
            _lib.check(L.fdb_vec_axpy(n, a, xb.device_ptr, yb.device_ptr))

    def scale(a, xv):
        for (n, _), xb in zip(sizes, blocks(xv)):
            _lib.check(L.fdb_vec_scale(n, a, xb.device_ptr))

    def copy(dst, src):
        for db, sb in zip(blocks(dst), blocks(src)):
            _lib.check(L.fdb_memcpy_d2d(db.device_ptr, sb.device_ptr, sb.nbytes))

    def touched(v):
        _touched(*blocks(v))

    def residual(r):
        """r = b - A x, returns ||r||"""
        A.mult(x, w)
        copy(r, b)
        axpy(-1.0, w, r)
        touched(r)
        return float(np.sqrt(dot(r, r)))

    beta = residual(Vs[0])
    hist = [beta]
    tol = max(rtol * beta, atol)
    it = 0
    while beta > tol and it < maxit:
        scale(1.0 / beta, Vs[0])
        touched(Vs[0])
        H = np.zeros((m + 1, m))
        cs, sn = np.zeros(m), np.zeros(m)
        g = np.zeros(m + 1)
        g[0] = beta
        k = 0
        for j in range(m):
            if M is not None:
                Zs[j].zero()
                for zb in blocks(Zs[j]):
                    zb.device_ptr
                M(Vs[j], Zs[j])
            A.mult(Zs[j], w)
            for i in range(j + 1):                      # modified Gram-Schmidt
                H[i, j] = dot(w, Vs[i])
                axpy(-H[i, j], Vs[i], w)
            touched(w)
            H[j + 1, j] = np.sqrt(max(dot(w, w), 0.0))
            if H[j + 1, j] > 0.0:
                copy(Vs[j + 1], w)
                scale(1.0 / H[j + 1, j], Vs[j + 1])
                touched(Vs[j + 1])
            for i in range(j):                          # previous rotations on the new column
                t = cs[i] * H[i, j] + sn[i] * H[i + 1, j]
                H[i + 1, j] = -sn[i] * H[i, j] + cs[i] * H[i + 1, j]
                H[i, j] = t
            r = np.hypot(H[j, j], H[j + 1, j])
            cs[j], sn[j] = (H[j, j] / r, H[j + 1, j] / r) if r > 0.0 else (1.0, 0.0)
            H[j, j] = r
            H[j + 1, j] = 0.0
            g[j + 1] = -sn[j] * g[j]
            g[j] = cs[j] * g[j]
            k = j + 1
            it += 1
            hist.append(abs(g[j + 1]))
            if abs(g[j + 1]) <= tol or it >= maxit or r == 0.0:
                break
        # x += Z y, R y = g (upper triangular k x k)
        y = np.zeros(k)
        for i in range(k - 1, -1, -1):
            y[i] = (g[i] - H[i, i + 1:k] @ y[i + 1:k]) / H[i, i] if H[i, i] != 0.0 else 0.0
        for i in range(k):
            axpy(y[i], Zs[i], x)
        touched(x)
        beta = residual(Vs[0])                          # the true residual at every restart
        hist[-1] = beta
    return it, hist


_PMG_KEYS = {"pmg_mg_coarse_degree": 1,
             "pmg_mg_levels_ksp_type": "chebyshev", "pmg_mg_levels_ksp_max_it": 2, "pmg_mg_levels_pc_type": "jacobi",
             "pmg_mg_levels_ksp_chebyshev_esteig": "0,0.1,0,1.1",
             "pmg_mg_coarse_ksp_type": "cg", "pmg_mg_coarse_pc_type": "jacobi", "pmg_mg_coarse_ksp_rtol": 1e-3,
             "pmg_mg_coarse_ksp_max_it": 500}


def pmg_options(sp):
    """The p-multigrid settings of ``solver_parameters`` with ``pc_type "python"``: ``pc_python_type``
    "firedrake.PMGPC" (halve the degree) or "firedrake.P1PC" (straight to the coarse degree), and the ``pmg_*`` keys of
    ``_PMG_KEYS`` with their defaults.  Nested dicts (``"pmg_mg_levels": {...}``, ``"pmg_mg_coarse": {...}``) are
    flattened as Firedrake does; any other ``pmg_*`` key is refused by name."""
    kind = sp.get("pc_python_type")
    if kind not in ("firedrake.PMGPC", "firedrake.P1PC"):
        raise NotImplementedError(f"pc_python_type {kind!r}: 'firedrake.PMGPC' or 'firedrake.P1PC'")
    flat = {}
    for k, v in sp.items():
        if isinstance(v, dict) and k.startswith("pmg_"):
            flat.update({f"{k}_{kk}": vv for kk, vv in v.items()})
        elif k.startswith("pmg_"):
            flat[k] = v
    bad = sorted(k for k in flat if k not in _PMG_KEYS)
    if bad:
        raise NotImplementedError(f"unknown p-multigrid option(s) {', '.join(bad)}: the supported ones are "
                                  f"{', '.join(_PMG_KEYS)}")
    o = dict(_PMG_KEYS, **flat)
    if o["pmg_mg_levels_pc_type"] != "jacobi":
        raise NotImplementedError(f"pmg_mg_levels_pc_type {o['pmg_mg_levels_pc_type']!r}: the level smoothers are "
                                  f"Jacobi-preconditioned ('jacobi')")
    o["halve"] = kind == "firedrake.PMGPC"
    return o


def _pmg(V, make, sp, bcs, hierarchy, allreduce, kappa=None, omega=0.8):
    """The :class:`mg.PMG` of the ``pc_type "python"`` options (:func:`pmg_options`) for the level forms ``make``."""
    from . import mg as _mg
    o = pmg_options(sp)
    est = tuple(float(v) for v in str(o["pmg_mg_levels_ksp_chebyshev_esteig"]).split(","))
    return _mg.PMG(V, make, bc_domains=tuple(s for bc in bcs for s in bc.sub_domains),
                   coarse_degree=int(o["pmg_mg_coarse_degree"]), halve=o["halve"], kappa=kappa,
                   smoother=o["pmg_mg_levels_ksp_type"], nu=int(o["pmg_mg_levels_ksp_max_it"]), omega=omega,
                   esteig=est, coarse_ksp=o["pmg_mg_coarse_ksp_type"], coarse_pc=o["pmg_mg_coarse_pc_type"],
                   coarse_rtol=float(o["pmg_mg_coarse_ksp_rtol"]), coarse_maxit=int(o["pmg_mg_coarse_ksp_max_it"]),
                   hierarchy=hierarchy, allreduce=allreduce)


def solve_nonlinear(F, L: op2.Dat, u: op2.Dat, bcs=(), solver_parameters=None, hierarchy=None, allreduce=None,
                    nullspace=None):
    """``solve(F == 0, u, bcs=bcs, solver_parameters=...)`` for nonlinear diffusion (``F`` a
    :class:`NonlinearDiffusion`) or hyperelasticity (a :class:`HyperElasticity` on a vector space) with the
    source ``L`` (the assembled right-hand side, e.g. ``assemble(mass(V), u=f)``): Newton's method with the
    full step (``snes_type newtonls``, ``snes_linesearch_type basic``) on the residual R(u) = F(u) - L,
    each step solved by GMRES with the exact Jacobian ``F.jacobian(u)``.  ``u`` is the initial guess
    and is overwritten with the solution.

    The Dirichlet values are applied to u first; the residual's rows on constrained nodes are zeroed
    and the Newton update vanishes there.  ``solver_parameters``: ``snes_rtol`` (1e-8), ``snes_atol``
    (1e-50), ``snes_max_it`` (50); ``ksp_type`` "gmres", ``ksp_gmres_restart`` (30), ``ksp_rtol``
    (1e-5), ``ksp_max_it`` (10000); ``mat_type`` "matfree" (default) | "aij"; ``pc_type`` "none"
    (default) | "jacobi" (the Jacobian's exact diagonal) | "mg" (needs ``hierarchy``; nonlinear
    diffusion: a V-cycle of the SPD operator ``Form(V, alpha, beta, kappa=D(u))``, rebuilt at every
    Newton step; hyperelasticity: a V-cycle of ``Elasticity(V, mu, lmbda, beta)``, the Jacobian at u = 0,
    built once per solve, with Jacobi smoothing damped by 0.6 as in :func:`solve`) | "python" (p-multigrid,
    :func:`pmg_options`, of the same operators).
    Converged when ||R(u)|| <= max(snes_rtol * ||R(u_0)||, snes_atol).  For hyperelasticity a
    non-finite residual norm (an inverted element: ln J of J <= 0) ends the solve with a
    :class:`ConvergenceError` whose reason is "DIVERGED_FNORM_NAN".  Returns (Newton residual norms,
    Krylov iterations per Newton step).

    Navier-Stokes (``F`` a :class:`NavierStokes`): ``L`` and ``u`` are MixedDats (velocity, pressure), the
    Dirichlet conditions are on the velocity, and the residual norm runs over both blocks.  Each step is
    matrix-free GMRES on ``F.jacobian(u)`` with the options of :func:`_solve_stokes`: ``mat_type`` "matfree",
    ``pc_type`` "none" (default) or "fieldsplit" (schur, diag / lower / upper; ``fieldsplit_0_pc_type`` "jacobi" or "mg" on
    ``Form(W, nu, beta)`` per component, ``fieldsplit_1_pc_type`` "jacobi", the pressure mass over nu), built
    once per solve.  ``nullspace`` "constant" removes the pressure mean from the residual, from every
    preconditioned vector and from the final pressure.  A non-finite residual norm ends the solve with a
    :class:`ConvergenceError` ("DIVERGED_FNORM_NAN").  The other forms take no ``nullspace``."""
    from . import _lib
    from . import mg as _mg
    if isinstance(F, NavierStokes):
        return _solve_navier_stokes(F, L, u, bcs, solver_parameters, hierarchy, nullspace)
    if nullspace is not None:
        raise NotImplementedError("nullspace is implemented for Navier-Stokes forms only")
    sp = {"snes_rtol": 1e-8, "snes_atol": 1e-50, "snes_max_it": 50, "ksp_type": "gmres",
          "ksp_gmres_restart": 30, "ksp_rtol": 1e-5, "ksp_max_it": 10000, "mat_type": "matfree",
          "pc_type": "none"}
    sp.update(solver_parameters or {})
    if sp["ksp_type"] != "gmres":
        raise NotImplementedError("ksp_type gmres only (a Newton Jacobian need not be symmetric or definite)")
    if sp["mat_type"] not in ("matfree", "aij"):
        raise NotImplementedError(f"mat_type {sp['mat_type']!r}")
    V = F.V
    bcs = tuple(bcs)
    lib = _lib.lib()
    n = L._data.size
    n_owned = L.dataset.set.size * L.cdim
    u.device_ptr
    for bc in bcs:
        bc.apply(u)
    R, du = V.dat(), V.dat()
    res = OneFormAssembler(F, u)

    def residual():
        import ctypes as C
        res.assemble(tensor=R)
        R.axpy(-1.0, L)
        for bc in bcs:
            bc.zero(R)
        out = C.c_double()
        _lib.check(lib.fdb_vec_dot(n_owned, R.device_ptr, R.device_ptr, C.byref(out)))
        return float(np.sqrt(allreduce(out.value) if allreduce else out.value))

    hyper = isinstance(F, HyperElasticity)

    def check_finite():
        if hyper and not np.isfinite(hist[-1]):
            raise ConvergenceError(f"nonlinear solve diverged: the residual norm is {hist[-1]} after "
                                   f"{len(kits)} Newton steps (DIVERGED_FNORM_NAN; an inverted element "
                                   f"has det F <= 0)", "DIVERGED_FNORM_NAN")

    hist = [residual()]
    kits = []
    check_finite()
    tol = max(sp["snes_rtol"] * hist[0], sp["snes_atol"])
    # J reads u in place: the matrix-free operator and the diagonal's context follow every update,
    # an assembled matrix is assembled again at every step
    J = F.jacobian(u)
    pc = sp["pc_type"]
    A = ctx = None
    d = V.dat() if pc == "jacobi" else None
    vc = None
    while hist[-1] > tol and len(kits) < sp["snes_max_it"]:
        if A is None or sp["mat_type"] != "matfree":
            A = assemble(J, bcs=bcs, mat_type=sp["mat_type"])
        if pc == "none":
            M = None
        elif pc == "jacobi":
            if ctx is None:
                ctx = A if isinstance(A, ImplicitMatrixContext) else ImplicitMatrixContext(J, bcs)
            ctx.getDiagonal(d)
            op2.par_loop(_mg.reciprocal_kernel(V.cdim), V.node_set, d(op2.RW))

            def M(r, z, d=d):
                _lib.check(lib.fdb_vec_pointwise_mult(n, r.device_ptr, d.device_ptr, z.device_ptr))
                z._device_written()
        elif pc == "mg":
            if hierarchy is None:
                raise ValueError("pc_type mg needs the mesh hierarchy")
            domains = tuple(s for bc in bcs for s in bc.sub_domains)
            if hyper:
                # J(0) = Elasticity: the same operator at every Newton step, so one V-cycle per solve
                if vc is None:
                    vc = _mg.VCycle(hierarchy, V.degree, lambda W, k=None: Elasticity(W, F.mu, F.lmbda, F.beta, F.ds),
                                    bc_domains=domains, allreduce=allreduce, cdim=3, omega=0.6)
            else:
                kap = F.diffusivity(u)
                vc = _mg.VCycle(hierarchy, V.degree, lambda W, k=None: Form(W, F.alpha, F.beta, k, F.ds),
                                bc_domains=domains, allreduce=allreduce, kappa=kap)
            top = len(hierarchy) - 1
            M = lambda r, z, vc=vc: vc.apply(top, r, z)
        elif pc == "python":
            # p-multigrid with the level forms of the "mg" branch: J(0) = Elasticity once per solve for
            # hyperelasticity, Form(V, alpha, beta, kappa=D(u)) at every Newton step for nonlinear diffusion
            if hyper:
                if vc is None:
                    vc = _pmg(V, lambda W, k=None: Elasticity(W, F.mu, F.lmbda, F.beta, F.ds), sp, bcs, hierarchy,
                              allreduce, omega=0.6)
            else:
                vc = _pmg(V, lambda W, k=None: Form(W, F.alpha, F.beta, k, F.ds), sp, bcs, hierarchy, allreduce,
                          kappa=F.diffusivity(u))
            M = lambda r, z, vc=vc: vc.apply(vc.top, r, z)
        else:
            raise NotImplementedError(f"pc_type {pc!r}")
        du.zero()
        du.device_ptr
        its, _ = gmres(A, R, du, M, rtol=sp["ksp_rtol"], restart=sp["ksp_gmres_restart"],
                       maxit=sp["ksp_max_it"], allreduce=allreduce)
        for bc in bcs:
            bc.zero(du)
        u.axpy(-1.0, du)
        kits.append(its)
        hist.append(residual())
        check_finite()
    return hist, kits


def solve(form: Form, L: op2.Dat, u: op2.Dat, bcs=(), solver_parameters=None, hierarchy=None, allreduce=None,
          nullspace=None):
    """``solve(a == L, u, bcs=bcs, solver_parameters=...)`` for the supported forms
    (firedrake/solving.py:128-260 -> LinearVariationalSolver; SURVEY.md section 3.5): assemble the
    operator, lift the Dirichlet values, run the Krylov solver on the device.  ``form``: a
    :class:`Form`, an :class:`Elasticity` form (vector space; Dirichlet values on every component) or an
    :class:`AdvectionDiffusion` form.

    ``L``: the assembled right-hand side (a Dat, e.g. ``assemble(mass(V), u=f)``).
    ``solver_parameters`` (PETSc option names, the subset that makes sense here):
    ``mat_type`` "matfree" (default) | "aij" | "is"; ``ksp_type`` "cg" (the default for symmetric forms) |
    "gmres" (:func:`gmres`, right-preconditioned and flexible; the default for nonsymmetric forms, which
    cg refuses), ``ksp_gmres_restart`` (30); ``pc_type`` "none" (default) | "jacobi" | "mg" (needs
    ``hierarchy``, a mg.MeshHierarchy whose finest mesh is ``form.V.mesh``; for advection-diffusion a
    V-cycle of its symmetric part ``Form(W, alpha, beta)``) | "python" with ``pc_python_type``
    "firedrake.PMGPC" or "firedrake.P1PC" (p-multigrid on ``V.mesh``, :class:`mg.PMG`, with the level forms of
    "mg" and the ``pmg_*`` options of :func:`pmg_options`; CG2 and CG3); ``ksp_rtol`` (1e-8), ``ksp_max_it`` (1000).
    A :class:`Stokes` form takes MixedDats and its own options (:func:`_solve_stokes`), and the only form
    that takes ``nullspace``.  Returns (iterations, residual history)."""
    from . import _lib
    if isinstance(form, Stokes):
        return _solve_stokes(form, L, u, bcs, solver_parameters, hierarchy, nullspace)
    if nullspace is not None:
        raise NotImplementedError("nullspace is implemented for Stokes forms only")
    symmetric = getattr(form, "symmetric", True)
    sp = {"mat_type": "matfree", "ksp_type": "cg" if symmetric else "gmres", "pc_type": "none", "ksp_rtol": 1e-8,
          "ksp_max_it": 1000, "ksp_gmres_restart": 30}
    sp.update(solver_parameters or {})
    if sp["ksp_type"] not in ("cg", "gmres"):
        raise NotImplementedError(f"ksp_type {sp['ksp_type']!r}: cg or gmres")
    if sp["ksp_type"] == "cg" and not symmetric:
        raise ValueError(f"ksp_type cg needs a symmetric operator, and {type(form).__name__} is not: use gmres")
    if isinstance(form, SpectralForm):
        if sp["mat_type"] != "matfree":
            raise NotImplementedError(f"mat_type {sp['mat_type']!r}: SpectralForm has no assembled matrix (there is "
                                      f"no assembled SEM matrix); use mat_type 'matfree'")
        if sp["pc_type"] not in ("none", "jacobi"):
            what = {"mg": "geometric multigrid", "python": "p-multigrid (PMGPC / P1PC)"}.get(sp["pc_type"], "it")
            raise NotImplementedError(f"pc_type {sp['pc_type']!r} on a SpectralForm: 'none' or 'jacobi' ({what} is "
                                      f"not implemented for the SEM operator)")
    V = form.V
    bcs = tuple(bcs)
    if getattr(V, "family", "CG") == "DQ":
        if bcs:
            raise ValueError("a DQ space takes no DirichletBC: impose the condition weakly "
                             "(InteriorPenalty(..., weak_bcs=...) and nitsche_load)")
        if sp["pc_type"] not in ("none", "jacobi"):
            raise NotImplementedError(f"pc_type {sp['pc_type']!r} on a DQ space: 'none' or 'jacobi' (there is no "
                                      f"DQ multigrid)")
        if sp["pc_type"] == "jacobi" and not (isinstance(form, DGTransport) and not (form.alpha or form.beta)):
            _dq_diagonal_kernel(V, 1.0, 0.0)          # refuses DQ4 before anything is assembled
    lib = _lib.lib()
    n = L._data.size
    # lifting (firedrake/assemble.py:1243-1254 + linear solver's rhs): u = g on the constrained nodes,
    # solve A (u - g) = L - K g on the free rows with homogeneous conditions
    g = V.dat()
    g.device_ptr
    for bc in bcs:
        bc.apply(g)
    lift = any(not (np.isscalar(bc.g) and bc.g == 0.0) for bc in bcs)
    b = V.dat()
    L.copy(b)
    if lift:
        Kg = OneFormAssembler(form, g, ()).assemble()
        b.axpy(-1.0, Kg)
    for bc in bcs:
        bc.zero(b)
    A = assemble(form, bcs=bcs, mat_type=sp["mat_type"])
    u.zero()
    u.device_ptr
    pc = sp["pc_type"]
    M = None
    if pc != "none":
        from . import mg as _mg
        if pc == "jacobi":
            ctx = A if isinstance(A, ImplicitMatrixContext) else ImplicitMatrixContext(form, bcs)
            d = ctx.getDiagonal(V.dat())
            op2.par_loop(_mg.reciprocal_kernel(V.cdim), V.node_set, d(op2.RW))

            def M(r, z):
                _lib.check(lib.fdb_vec_pointwise_mult(n, r.device_ptr, d.device_ptr, z.device_ptr))
                z._device_written()
        elif pc == "mg":
            if hierarchy is None:
                raise ValueError("pc_type mg needs the mesh hierarchy")
            # with a coefficient field, every coarser level gets the injection of the next finer
            # level's kappa (VCycle's ``kappa``), as Firedrake coarsens coefficients for rediscretised
            # multigrid
            # elasticity: the Jacobi smoother's damping is 0.6, not 0.8.  The spectrum of D^-1 A of the coupled
            # operator reaches past 2 / 0.8, so 0.8 amplifies its highest modes: CG1 at nu = 0.3 took 16 and
            # 97 iterations on 8^3 and 16^3 with 0.8, 8 and 9 with 0.6 (DESIGN.md section 4.8)
            # advection-diffusion: a V-cycle of its symmetric part Form(W, alpha, beta) on every level (the
            # convective term is left to the outer GMRES, DESIGN.md section 4.10)
            # boundary terms: the same (gamma, sub_domain) pairs on every level (the names are mesh-level)
            ds = getattr(form, "ds", ())
            if isinstance(form, Elasticity):
                make = lambda W, k=None: Elasticity(W, form.mu, form.lmbda, form.beta, ds)
                omega = 0.6
            else:
                make = lambda W, k=None: Form(W, form.alpha, form.beta, k, ds)
                omega = 0.8
            vc = _mg.VCycle(hierarchy, V.degree, make,
                            bc_domains=tuple(s for bc in bcs for s in bc.sub_domains), allreduce=allreduce,
                            kappa=getattr(form, "kappa", None), cdim=V.cdim, omega=omega)
            top = len(hierarchy) - 1
            M = lambda r, z: vc.apply(top, r, z)
        elif pc == "python":
            # p-multigrid (firedrake.PMGPC / P1PC) with the level forms and Jacobi damping of the "mg" branch
            ds = getattr(form, "ds", ())
            if isinstance(form, Elasticity):
                make, omega = (lambda W, k=None: Elasticity(W, form.mu, form.lmbda, form.beta, ds)), 0.6
            else:
                make, omega = (lambda W, k=None: Form(W, form.alpha, form.beta, k, ds)), 0.8
            pm = _pmg(V, make, sp, bcs, hierarchy, allreduce, kappa=getattr(form, "kappa", None), omega=omega)
            M = lambda r, z: pm.apply(pm.top, r, z)
        else:
            raise NotImplementedError(f"pc_type {pc!r}")
    if sp["ksp_type"] == "gmres":
        its, hist = gmres(A, b, u, M, rtol=sp["ksp_rtol"], restart=sp["ksp_gmres_restart"], maxit=sp["ksp_max_it"],
                          allreduce=allreduce)
    elif M is None:
        its, hist = cg(A, b, u, rtol=sp["ksp_rtol"], maxit=sp["ksp_max_it"], allreduce=allreduce)
    else:
        its, hist = _mg.pcg(A, b, u, M, rtol=sp["ksp_rtol"], maxit=sp["ksp_max_it"], allreduce=allreduce)
    if lift:
        u.axpy(1.0, g)
    else:
        for bc in bcs:
            bc.apply(u)
    return its, hist


def _solve_stokes(form: Stokes, L: op2.MixedDat, up: op2.MixedDat, bcs=(), solver_parameters=None,
                  hierarchy=None, nullspace=None):
    """``solve(a == L, up, bcs=bcs, solver_parameters=..., nullspace=...)`` for :class:`Stokes`, with the option
    names of Firedrake's matrix-free Stokes demo:

    - ``mat_type`` "matfree" (the only one); ``ksp_type`` "gmres" (default; "cg" is refused, the operator is
      indefinite), ``ksp_gmres_restart`` (30), ``ksp_rtol`` (1e-8), ``ksp_max_it`` (1000).
    - ``pc_type`` "none" (default) or "fieldsplit" with ``pc_fieldsplit_type`` "schur" and
      ``pc_fieldsplit_schur_fact_type`` "diag": z_u = P_0(r_u), z_p = P_1(r_p); "lower" or "upper": PETSc's
      block-triangular factorisations with S^-1 ~ -P_1, one extra Stokes action per application
      (:func:`_schur_factorisation`).
      ``fieldsplit_0_pc_type`` "jacobi" (default: the inverse diagonal of the velocity block) or "mg" (one
      V-cycle of ``Form(W, mu, beta)`` on the vector spaces of ``hierarchy``, with the velocity conditions'
      sub-domains); ``fieldsplit_1_pc_type`` "jacobi" (default): the inverse diagonal of the Schur complement
      approximation (1/mu) M_p, as Firedrake's MassInvPC with the viscosity.  Only one application of each
      (``fieldsplit_*_ksp_type`` "preonly").
    - ``nullspace`` "constant": the pressure is determined up to a constant
      (``MixedVectorSpaceBasis(Z, [Z.sub(0), VectorSpaceBasis(constant=True)])``).  The dof-mean of the
      pressure block is removed from the right-hand side, from every preconditioned vector and from the
      final pressure.

    Dirichlet conditions are on the velocity; their values are lifted with the full Stokes action on
    (g, 0), so the pressure rows receive -q div g.  ``up`` is overwritten with the solution.  Returns
    (iterations, residual history)."""
    sp = {"mat_type": "matfree", "ksp_type": "gmres", "pc_type": "none", "ksp_rtol": 1e-8, "ksp_max_it": 1000,
          "ksp_gmres_restart": 30, "fieldsplit_0_pc_type": "jacobi", "fieldsplit_1_pc_type": "jacobi",
          "fieldsplit_0_ksp_type": "preonly", "fieldsplit_1_ksp_type": "preonly"}
    sp.update(solver_parameters or {})
    if sp["ksp_type"] == "cg":
        raise ValueError("ksp_type cg needs a positive definite operator, and the Stokes operator is indefinite: "
                         "use gmres")
    if sp["ksp_type"] != "gmres":
        raise NotImplementedError(f"ksp_type {sp['ksp_type']!r}: Stokes solves with gmres")
    if sp["mat_type"] != "matfree":
        raise NotImplementedError(f"mat_type {sp['mat_type']!r}: Stokes has no assembled matrix, use mat_type "
                                  f"'matfree'")
    if nullspace not in (None, "constant"):
        raise NotImplementedError(f"nullspace {nullspace!r}: None or 'constant' (constant pressures)")
    _check_fieldsplit(sp, hierarchy)
    V, Q = form.V, form.Q
    bcs = tuple(bcs)
    remove_pressure_mean = _pressure_mean_remover(Q) if nullspace else None

    # lifting: A (up - (g, 0)) = L - A (g, 0) with homogeneous conditions
    g = form.dat()
    g.zero()
    g[0].device_ptr
    for bc in bcs:
        bc.apply(g[0])
    lift = any(not (np.isscalar(bc.g) and bc.g == 0.0) for bc in bcs)
    b = form.dat()
    L.copy(b)
    if lift:
        b.axpy(-1.0, StokesAssembler(form, g).assemble())
    for bc in bcs:
        bc.zero(b[0])
    if nullspace:
        remove_pressure_mean(b)
    A = StokesMatrixContext(form, bcs)
    up.zero()
    for d in up:
        d.device_ptr
    M = _fieldsplit_pc(V, Q, form.mu, form.beta, up, bcs, sp, hierarchy, remove_pressure_mean)
    its, hist = gmres(A, b, up, M, rtol=sp["ksp_rtol"], restart=sp["ksp_gmres_restart"], maxit=sp["ksp_max_it"])
    if nullspace:
        remove_pressure_mean(up)
    if lift:
        up[0].axpy(1.0, g[0])
    else:
        for bc in bcs:
            bc.apply(up[0])
    return its, hist


_SCHUR_FACTORISATIONS = ("diag", "lower", "upper")


def _check_fieldsplit(sp, hierarchy):
    """The preconditioner options of the Taylor-Hood solves (:func:`_solve_stokes`, Newton on
    :class:`NavierStokes`): ``pc_type`` "none" or the Schur fieldsplit, factorised "diag", "lower" or "upper"."""
    pc = sp["pc_type"]
    if pc not in ("none", "fieldsplit"):
        raise NotImplementedError(f"pc_type {pc!r}: 'none' or 'fieldsplit'")
    if pc == "fieldsplit":
        if sp.get("pc_fieldsplit_type") != "schur":
            raise NotImplementedError(f"pc_fieldsplit_type {sp.get('pc_fieldsplit_type')!r}: 'schur' only")
        if sp.get("pc_fieldsplit_schur_fact_type") not in _SCHUR_FACTORISATIONS:
            raise NotImplementedError(f"pc_fieldsplit_schur_fact_type {sp.get('pc_fieldsplit_schur_fact_type')!r}: "
                                      f"not built ('diag' only, or 'lower' / 'upper')")
        for f in ("0", "1"):
            if sp[f"fieldsplit_{f}_ksp_type"] != "preonly":
                raise NotImplementedError(f"fieldsplit_{f}_ksp_type {sp[f'fieldsplit_{f}_ksp_type']!r}: 'preonly' "
                                          f"only")
        if sp["fieldsplit_0_pc_type"] not in ("jacobi", "mg"):
            raise NotImplementedError(f"fieldsplit_0_pc_type {sp['fieldsplit_0_pc_type']!r}: 'jacobi' or 'mg'")
        if sp["fieldsplit_1_pc_type"] != "jacobi":
            raise NotImplementedError(f"fieldsplit_1_pc_type {sp['fieldsplit_1_pc_type']!r}: 'jacobi' (the "
                                      f"inverse diagonal of the pressure mass matrix over mu)")
        if sp["fieldsplit_0_pc_type"] == "mg" and hierarchy is None:
            raise ValueError("fieldsplit_0_pc_type mg needs the mesh hierarchy")


def _pressure_mean_remover(Q):
    """v -> v with the dof-mean of its pressure block removed (the constant-pressure nullspace)."""
    ones = Q.dat(np.ones(Q.node_count))

    def remove_pressure_mean(v):
        v[1].axpy(-v[1].inner(ones) / Q.node_count, ones)
    return remove_pressure_mean


def _fieldsplit_pc(V, Q, mu, beta, up, bcs, sp, hierarchy, remove_pressure_mean=None):
    """The preconditioner ``M(r, z)`` of the Taylor-Hood GMRES solves (None: none), from the options that
    :func:`_check_fieldsplit` accepted.  The Schur fieldsplit preconditions the velocity with Jacobi or one
    V-cycle per component of ``Form(W, mu, beta)`` and the pressure with the inverse diagonal of (1/mu) M_p,
    combined "diag" or as the "lower" / "upper" factorisation (:func:`_schur_factorisation`).  It does not
    depend on the velocity, so one is built per solve.  ``remove_pressure_mean`` (the constant nullspace) is
    applied to every preconditioned vector."""
    from . import _lib
    from . import mg as _mg
    lib = _lib.lib()
    nullspace = remove_pressure_mean is not None
    M = None
    if sp["pc_type"] == "fieldsplit":
        n_u, n_p = up[0]._data.size, up[1]._data.size
        # pressure: the inverse diagonal of (1/mu) M_p
        dp = ImplicitMatrixContext(Form(Q, 0.0, 1.0 / mu)).getDiagonal(Q.dat())
        op2.par_loop(_mg.reciprocal_kernel(1), Q.node_set, dp(op2.RW))
        if sp["fieldsplit_0_pc_type"] == "jacobi":
            # the velocity block is mu * (vector Laplacian) + beta * mass: the scalar diagonal on every component
            Vs = FunctionSpace(V.mesh, V.degree)
            ds = ImplicitMatrixContext(Form(Vs, mu, beta)).getDiagonal(Vs.dat()).data_ro
            du = V.dat(np.repeat(ds, 3).reshape(-1, 3))
            for bc in bcs:
                bc.set(du, 1.0)
            op2.par_loop(_mg.reciprocal_kernel(3), V.node_set, du(op2.RW))

            def Mu(r, z):
                _lib.check(lib.fdb_vec_pointwise_mult(n_u, r.device_ptr, du.device_ptr, z.device_ptr))
                z._device_written()
        else:
            # the velocity block is three uncoupled copies of the scalar Form(W, mu, beta): one scalar V-cycle
            # per component (the Helmholtz diagonal kernel that the smoother needs is scalar)
            vc = _mg.VCycle(hierarchy, V.degree, lambda W, k=None: Form(W, mu, beta),
                            bc_domains=tuple(s for bc in bcs for s in bc.sub_domains))
            top = len(hierarchy) - 1
            nn = V.node_count
            comp = [op2.DeviceArray.from_host(np.ascontiguousarray(3 * np.arange(nn, dtype=np.int32) + c))
                    for c in range(3)]
            rs, zs = vc.spaces[-1].dat(), vc.spaces[-1].dat()

            def Mu(r, z):
                for c in range(3):
                    _lib.check(lib.fdb_vec_gather(nn, comp[c].ptr, r.device_ptr, rs.device_ptr))
                    _mg._touched(rs)
                    zs.zero()
                    zs.device_ptr
                    vc.apply(top, rs, zs)
                    _lib.check(lib.fdb_vec_scatter(nn, comp[c].ptr, zs.device_ptr, z.device_ptr))
                z._device_written()

        def Mp(r, z):
            _lib.check(lib.fdb_vec_pointwise_mult(n_p, r.device_ptr, dp.device_ptr, z.device_ptr))
            z._device_written()

        fact = sp["pc_fieldsplit_schur_fact_type"]
        if fact == "diag":
            def M(r, z):
                Mu(r[0], z[0])
                Mp(r[1], z[1])
                if nullspace:
                    remove_pressure_mean(z)
        else:
            # the off-diagonal blocks B and B^T do not depend on u, so the Stokes operator with the velocity
            # conditions applies them for both solves (cheaper than the Navier-Stokes Jacobian action)
            S = Stokes(V, Q, mu, beta)
            M = _schur_factorisation(fact, Mu, Mp, StokesMatrixContext(S, bcs), S.dat, remove_pressure_mean)
    elif nullspace:
        def M(r, z):
            r.copy(z)
            remove_pressure_mean(z)
    return M


def _schur_factorisation(fact, Mu, Mp, A, new, remove_pressure_mean=None):
    """``M(r, z)`` of the "lower" or "upper" Schur factorisation (PETSc's ``pc_fieldsplit_schur_fact_type``) of
    the Taylor-Hood operator A = [[F, B^T], [B, 0]], whose pressure rows are -q div u.  ``Mu(r_u, z_u)`` applies
    P_0 ~ F^-1 and ``Mp(r_p, z_p)`` applies P_1 ~ (B F^-1 B^T)^-1; the Schur complement is S = -B F^-1 B^T, so
    S^-1 ~ -P_1 (the "diag" factorisation applies +P_1, PETSc's schur_scale -1):

    - "lower", the inverse of [[F, 0], [B, S]]: z_u = P_0 r_u, then z_p = -P_1 (r_p - B z_u);
    - "upper", the inverse of [[F, B^T], [0, S]]: z_p = -P_1 r_p, then z_u = P_0 (r_u - B^T z_p).

    ``A.mult`` applies the operator with the velocity conditions: B z_u is the pressure block of A (z_u, 0) and
    B^T z_p the velocity block of A (0, z_p), zero on the constrained rows.  One extra action of A per
    application.  ``new()`` makes a MixedDat of the two spaces for the work vectors.  ``remove_pressure_mean``
    (the constant nullspace) is applied to every preconditioned vector."""
    from . import _lib
    lib = _lib.lib()
    w, y = new(), new()

    def negate(v):
        _lib.check(lib.fdb_vec_scale(v._data.size, -1.0, v.device_ptr))
        v._device_written()

    def M(r, z):
        if fact == "lower":
            Mu(r[0], z[0])
            z[0].copy(w[0])
            w[1].zero()
            A.mult(w, y)
            r[1].copy(w[1])
            w[1].axpy(-1.0, y[1])
            Mp(w[1], z[1])
            negate(z[1])
        else:
            Mp(r[1], z[1])
            negate(z[1])
            w[0].zero()
            z[1].copy(w[1])
            A.mult(w, y)
            r[0].copy(w[0])
            w[0].axpy(-1.0, y[0])
            Mu(w[0], z[0])
        if remove_pressure_mean is not None:
            remove_pressure_mean(z)
    return M


def _solve_navier_stokes(F: NavierStokes, L: op2.MixedDat, up: op2.MixedDat, bcs=(), solver_parameters=None,
                         hierarchy=None, nullspace=None):
    """Newton's method for :class:`NavierStokes` (``snes_type newtonls``, ``snes_linesearch_type basic``) on
    R(up) = F(up) - L over MixedDats; see :func:`solve_nonlinear`."""
    sp = {"snes_rtol": 1e-8, "snes_atol": 1e-50, "snes_max_it": 50, "ksp_type": "gmres",
          "ksp_gmres_restart": 30, "ksp_rtol": 1e-5, "ksp_max_it": 10000, "mat_type": "matfree",
          "pc_type": "none", "fieldsplit_0_pc_type": "jacobi", "fieldsplit_1_pc_type": "jacobi",
          "fieldsplit_0_ksp_type": "preonly", "fieldsplit_1_ksp_type": "preonly"}
    sp.update(solver_parameters or {})
    if sp["ksp_type"] != "gmres":
        raise NotImplementedError(f"ksp_type {sp['ksp_type']!r}: the Navier-Stokes Jacobian is nonsymmetric and "
                                  f"indefinite, Newton solves with gmres")
    if sp["mat_type"] != "matfree":
        raise NotImplementedError(f"mat_type {sp['mat_type']!r}: the Navier-Stokes Jacobian has no assembled "
                                  f"matrix, use mat_type 'matfree'")
    if nullspace not in (None, "constant"):
        raise NotImplementedError(f"nullspace {nullspace!r}: None or 'constant' (constant pressures)")
    _check_fieldsplit(sp, hierarchy)
    V, Q = F.V, F.Q
    bcs = tuple(bcs)
    remove_pressure_mean = _pressure_mean_remover(Q) if nullspace else None
    for d in up:
        d.device_ptr
    for bc in bcs:
        bc.apply(up[0])
    R, du = F.dat(), F.dat()
    res = StokesAssembler(F, up)

    def residual():
        res.assemble(tensor=R)
        R.axpy(-1.0, L)
        for bc in bcs:
            bc.zero(R[0])
        if nullspace:
            remove_pressure_mean(R)
        return R.norm()

    def check_finite():
        if not np.isfinite(hist[-1]):
            raise ConvergenceError(f"Newton diverged: the residual norm is {hist[-1]} after {len(kits)} steps "
                                   f"(DIVERGED_FNORM_NAN)", "DIVERGED_FNORM_NAN")

    hist = [residual()]
    kits = []
    check_finite()
    tol = max(sp["snes_rtol"] * hist[0], sp["snes_atol"])
    # J reads up[0] in place, so one matrix-free operator serves every step; the preconditioner does not
    # depend on u
    A = StokesMatrixContext(F.jacobian(up), bcs)
    M = _fieldsplit_pc(V, Q, F.nu, F.beta, up, bcs, sp, hierarchy, remove_pressure_mean)
    while hist[-1] > tol and len(kits) < sp["snes_max_it"]:
        du.zero()
        for d in du:
            d.device_ptr
        its, _ = gmres(A, R, du, M, rtol=sp["ksp_rtol"], restart=sp["ksp_gmres_restart"], maxit=sp["ksp_max_it"])
        for bc in bcs:
            bc.zero(du[0])
        up.axpy(-1.0, du)
        kits.append(its)
        hist.append(residual())
        check_finite()
    if nullspace:
        remove_pressure_mean(up)
    return hist, kits


class DGAdvection:
    """Right-hand side ``assemble(L1)`` of the DG advection demo (reference
    demos/DG_advection/DG_advection.py.rst:182-217) on a :class:`QuadMesh`.

    ``fused=False``: three parloops -- cells, exterior facets, interior facets --
    exactly the kernels ``OneFormAssembler`` would run
    (firedrake/assemble.py:1069-1096), with the reference's facet-kernel ABI.
    ``fused=True``: ONE owner-computes pass over the cells (each cell adds its
    cell term and the fluxes through its four facets into its own dofs): no
    atomics, deterministic, ~3x less traffic; the only off-cell data is the q of
    neighbouring cells, i.e. a ghost-cell halo when the mesh is a slab of a
    partitioned run (``halo`` = ``firedrake_b200.halo.Halo`` on the DQ dofs).
    """

    def __init__(self, mesh, dt, q_in=1.0, nq=3, fused=False, halo=None):
        self.mesh, self.fused = mesh, fused
        C_ = mesh.num_cells
        owned = mesh.num_owned_cells
        self.cell_set = op2.Set((owned, owned, C_))
        self.dq_nodes = op2.Set((4 * owned, 4 * owned, 4 * C_))
        self.dq_dset = op2.DataSet(self.dq_nodes, 1, halo=halo)
        self.vertices = op2.Set(mesh.node_count)
        dg, cg = mesh.dg1_map, mesh.coord_map
        self.cell_dq = op2.Map(self.cell_set, self.dq_nodes, 4, dg)
        self.cell_cg = op2.Map(self.cell_set, self.vertices, 4, cg)
        self.coordinates = op2.Dat(op2.DataSet(self.vertices, 2), mesh.coordinates)
        self.consts = op2.Global(2, [dt, q_in])
        self.nq = nq
        self._loops = None
        if fused:
            self.nbr = op2.Dat(op2.DataSet(self.cell_set, 4), mesh.nbr, dtype=np.int32)
            self.nbr_facet = op2.Dat(op2.DataSet(self.cell_set, 4), mesh.nbr_facet, dtype=np.uint32)
            return
        if halo is not None:
            raise NotImplementedError("the facet-loop form runs unpartitioned; use fused=True")
        self.ext_set = op2.Set(len(mesh.ext_facet_cells))
        self.int_set = op2.Set(len(mesh.int_facet_cells))
        # facet->node maps: the nodes of cell '+' then of cell '-'
        # (firedrake/cython/dmcommon.pyx:1636-1677)
        self.ext_dq = op2.Map(self.ext_set, self.dq_nodes, 4, dg[mesh.ext_facet_cells])
        self.ext_cg = op2.Map(self.ext_set, self.vertices, 4, cg[mesh.ext_facet_cells])
        ic = mesh.int_facet_cells
        self.int_dq = op2.Map(self.int_set, self.dq_nodes, 8, np.concatenate([dg[ic[:, 0]], dg[ic[:, 1]]], axis=1))
        self.int_cg = op2.Map(self.int_set, self.vertices, 8, np.concatenate([cg[ic[:, 0]], cg[ic[:, 1]]], axis=1))
        self.ext_facet = op2.Dat(op2.DataSet(self.ext_set, 1), mesh.ext_facet_local, dtype=np.uint32)
        self.int_facet = op2.Dat(op2.DataSet(self.int_set, 2), mesh.int_facet_local, dtype=np.uint32)

    def function(self, data=None):
        return op2.Dat(self.dq_dset, data)

    def velocity(self, data):
        return op2.Dat(op2.DataSet(self.vertices, 2), data)

    def assemble(self, q, u, tensor=None):
        if tensor is None:
            tensor = self.function()
        key = (id(q), id(u), id(tensor))
        if self._loops is None or self._key != key:
            self._key = key
            mk = lambda integral: op2.Kernel("dg_advection", degree=1, integral=integral, nq=self.nq)
            X, G = self.coordinates, self.consts
            gk = lambda k, maps: op2.GlobalKernel(k, maps, extruded=False)
            if self.fused:
                self._loops = [
                    op2.Parloop(gk(mk("fused"), [self.cell_dq, self.cell_cg]), self.cell_set,
                                [tensor(op2.INC, self.cell_dq), X(op2.READ, self.cell_cg),
                                 q(op2.READ, self.cell_dq), u(op2.READ, self.cell_cg), G(op2.READ),
                                 self.nbr_facet(op2.READ), self.nbr(op2.READ)])]
            else:
                self._loops = [
                    op2.Parloop(gk(mk("cell"), [self.cell_dq, self.cell_cg]), self.cell_set,
                                [tensor(op2.INC, self.cell_dq), X(op2.READ, self.cell_cg), q(op2.READ, self.cell_dq),
                                 u(op2.READ, self.cell_cg), G(op2.READ)]),
                    op2.Parloop(gk(mk("exterior_facet"), [self.ext_dq, self.ext_cg]), self.ext_set,
                                [tensor(op2.INC, self.ext_dq), X(op2.READ, self.ext_cg), q(op2.READ, self.ext_dq),
                                 u(op2.READ, self.ext_cg), G(op2.READ), self.ext_facet(op2.READ)]),
                    op2.Parloop(gk(mk("interior_facet"), [self.int_dq, self.int_cg]), self.int_set,
                                [tensor(op2.INC, self.int_dq), X(op2.READ, self.int_cg), q(op2.READ, self.int_dq),
                                 u(op2.READ, self.int_cg), G(op2.READ), self.int_facet(op2.READ)]),
                ]
        tensor.zero()
        if self.fused and q.dataset.halo is not None and not q.halo_valid:
            # ghost-cell q must be current before ANY cell runs (every cell may border a ghost)
            q.dataset.halo.global_to_local_begin(q)
            q.dataset.halo.global_to_local_end(q)
        tensor.frozen_halo = True          # owner-computes: nothing to send back
        for loop in self._loops:
            loop()
        tensor.frozen_halo = False
        return tensor


def dg_slab(nx, ny, rank, nranks):
    """Slab of the nx x ny quad mesh for ``rank`` with ghost-cell columns, and
    the (rank, send, recv) halo lists of its DQ1 dofs."""
    from .partition import slab_bounds
    from .utility_meshes import QuadMesh
    x0, x1 = slab_bounds(nx, nranks, rank)
    mesh = QuadMesh(x1 - x0, ny, ix0=x0, nx_global=nx, ghost_left=rank > 0,
                    ghost_right=rank < nranks - 1)
    dofs = lambda cells: (np.asarray(cells)[:, None] * 4 + np.arange(4)[None, :]).ravel().astype(np.int32)
    neigh = []
    if rank > 0:
        neigh.append((rank - 1, dofs(mesh.first_owned_column), dofs(mesh.ghost_cells_left)))
    if rank < nranks - 1:
        neigh.append((rank + 1, dofs(mesh.last_owned_column), dofs(mesh.ghost_cells_right)))
    return mesh, neigh
