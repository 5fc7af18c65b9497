"""1-D element tabulation used to feed the element kernels.

The reference obtains these tables at run time from FIAT/FInAT (not present in
this image; SURVEY.md section 8c): the default CG variant on tensor-product
cells is "spectral" = Gauss-Lobatto-Legendre nodes
(reference docs/source/variational-problems.rst:286-301), DG on intervals uses
Gauss-Legendre nodes, and quadrature on tensor-product cells is a tensor
Gauss-Legendre rule.  Every kernel in this package takes the tables as RUNTIME
inputs (never baked constants), so a caller that does have FInAT can pass the
real ones.

1-D dof numbering is FIAT's entity ordering on the interval: dof 0 = left
vertex, dof 1 = right vertex, dofs 2.. = interior nodes left to right.
"""
from __future__ import annotations

import numpy as np
from numpy.polynomial import legendre as _leg

__all__ = ["gll_points", "gll_weights", "gauss_legendre", "Interval1D", "interval_element"]


def gauss_legendre(m: int):
    """m-point Gauss-Legendre rule on [0, 1] (exact to degree 2m-1)."""
    x, w = _leg.leggauss(m)
    return 0.5 * (x + 1.0), 0.5 * w


def gll_points(p: int) -> np.ndarray:
    """The p+1 Gauss-Lobatto-Legendre points on [0, 1], ascending."""
    if p < 1:
        raise ValueError("degree must be >= 1")
    if p == 1:
        return np.array([0.0, 1.0])
    c = np.zeros(p + 1)
    c[p] = 1.0
    dc = _leg.legder(c)
    r = np.sort(_leg.legroots(dc).real)
    # two Newton sweeps on P_p'(x) to polish the roots
    d2 = _leg.legder(dc)
    for _ in range(2):
        r = r - _leg.legval(r, dc) / _leg.legval(r, d2)
    x = np.concatenate([[-1.0], r, [1.0]])
    x = 0.5 * (x - x[::-1])          # enforce symmetry
    return 0.5 * (x + 1.0)


def gll_weights(p: int) -> np.ndarray:
    """The weights of the (p+1)-point Gauss-Lobatto-Legendre rule on [0, 1] at :func:`gll_points` (ascending),
    exact to degree 2p-1: w_i = 1 / (p (p+1) P_p(x_i)^2) with x_i on [-1, 1]."""
    x = 2.0 * gll_points(p) - 1.0
    c = np.zeros(p + 1)
    c[p] = 1.0
    return 1.0 / (p * (p + 1) * _leg.legval(x, c) ** 2)


def _lagrange_tab(nodes: np.ndarray, pts: np.ndarray):
    """Values and first derivatives of the Lagrange basis on ``nodes`` at ``pts``.

    Returns (B, D) with B[q, i] = l_i(pts[q]), D[q, i] = l_i'(pts[q]).
    """
    n = len(nodes)
    B = np.ones((len(pts), n))
    D = np.zeros((len(pts), n))
    for i in range(n):
        others = [j for j in range(n) if j != i]
        denom = np.prod([nodes[i] - nodes[j] for j in others])
        for q, x in enumerate(pts):
            B[q, i] = np.prod([x - nodes[j] for j in others]) / denom
            s = 0.0
            for k in others:
                s += np.prod([x - nodes[j] for j in others if j != k])
            D[q, i] = s / denom
    return B, D


class Interval1D:
    """A 1-D Lagrange element of degree p on [0,1] tabulated at a quadrature rule.

    Attributes
    ----------
    nodes : (p+1,) node positions in *dof numbering* (entity ordered)
    B, D  : (nq, p+1) basis values / derivatives at the quadrature points,
            columns in dof numbering
    xq, wq : quadrature points and weights on [0, 1]

    ``quadrature="gauss"`` (the default) tabulates at the nq-point Gauss-Legendre rule.  ``quadrature="gll"``
    tabulates at the p+1 Gauss-Lobatto-Legendre points of a "gll" element, in DOF order (xq = nodes): the rule is
    collocated with the nodes, so B is exactly the identity, D is the GLL differentiation matrix in dof numbering
    and the mass matrix integrated with the rule is diagonal (spectral-element mass lumping).
    """

    def __init__(self, degree: int, nq: int, variant: str = "gll", quadrature: str = "gauss"):
        self.degree = degree
        n = degree + 1
        if variant == "gll":
            pos = gll_points(degree)
        elif variant == "gl":
            pos, _ = gauss_legendre(n)
        elif variant == "equispaced":
            pos = np.linspace(0.0, 1.0, n)
        else:
            raise ValueError(f"unknown variant {variant!r}")
        self.variant = variant
        # entity ordering: vertices first, then interior (CG); DG (gl) has only
        # interior dofs, numbered left to right.
        if variant == "gl":
            order = np.arange(n)
        else:
            order = np.array([0, n - 1] + list(range(1, n - 1)))
        self.dof_to_pos = order                    # dof a sits at ascending position order[a]
        self.nodes = pos[order]
        self.quadrature = quadrature
        if quadrature == "gauss":
            self.xq, self.wq = gauss_legendre(nq)
            self.B, self.D = _lagrange_tab(self.nodes, self.xq)
        elif quadrature == "gll":
            if variant != "gll" or nq != n:
                raise ValueError(f"quadrature 'gll' is collocated with the nodes of a 'gll' element: nq = degree+1 "
                                 f"= {n} (got variant {variant!r}, nq {nq})")
            self.xq, self.wq = self.nodes.copy(), gll_weights(degree)[order]
            _, self.D = _lagrange_tab(self.nodes, self.xq)
            self.B = np.eye(n)                     # exactly: l_a(x_b) = delta_ab
        else:
            raise ValueError(f"unknown quadrature {quadrature!r}: 'gauss' or 'gll'")
        self.nq = nq
        self.ndof = n

    def tabulate(self, pts):
        return _lagrange_tab(self.nodes, np.asarray(pts, dtype=float))


_cache = {}


def interval_element(degree: int, nq: int | None = None, variant: str = "gll",
                     quadrature: str = "gauss") -> Interval1D:
    """Cached constructor.  ``nq`` defaults to degree+1 Gauss points, the rule
    SURVEY.md section 8(d) pins for Poisson/Helmholtz CGp (Firedrake side:
    ``dx(degree=2*p)``).  ``quadrature="gll"``: the GLL rule at the nodes, in dof order (Firedrake's
    ``dx(scheme=gauss_lobatto_legendre_cube_rule(...))``)."""
    if nq is None:
        nq = degree + 1
    key = (degree, nq, variant, quadrature)
    if key not in _cache:
        _cache[key] = Interval1D(degree, nq, variant, quadrature)
    return _cache[key]
