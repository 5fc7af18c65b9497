"""TEST INFRASTRUCTURE: the engine entry points that one ``solve`` calls, in order, with pc_type none, jacobi, mg and
the p-multigrid python options, on the p-multigrid mock engine (tests/test_pmg_host_mock.py).  The same function
recorded tests/golden/solve_pc_engine_calls.json from the version before FDMPC was added."""
import numpy as np

from test_pmg_host_mock import PMGEngine, pmg_mock

CASES = {
    "none": {"pc_type": "none"},
    "jacobi": {"pc_type": "jacobi"},
    "mg": {"pc_type": "mg"},
    "pmgpc": {"pc_type": "python", "pc_python_type": "firedrake.PMGPC"},
    "p1pc": {"pc_type": "python", "pc_python_type": "firedrake.P1PC"},
}


class Recorder(PMGEngine):
    """PMGEngine that also records the name of every engine entry point called."""

    def __init__(self, oracle):
        super().__init__(oracle)
        self.names = None

    def __getattribute__(self, name):
        if name.startswith("fdb_"):
            names = object.__getattribute__(self, "names")
            if names is not None:
                names.append(name)
        return object.__getattribute__(self, name)


class recording(pmg_mock):
    def __init__(self, oracle):
        self.engine = Recorder(oracle)


def solve_calls(oracle, case):
    """(entry-point names, PMGEngine trace) of one Poisson solve on CG2 over a warped 4^3 mesh, the finest of a
    two-level hierarchy, Dirichlet bottom and top, stopped after two iterations (the set-up and the repeating part of
    an iteration).  The trace entries are "name" or "name:n"."""
    from firedrake_b200 import mg
    from firedrake_b200.assemble import DirichletBC, Form, FunctionSpace, assemble, mass, solve
    with recording(oracle) as eng:
        h = mg.MeshHierarchy(2, 2, 2, 1, warp=0.05)
        V = FunctionSpace(h[1], 2)
        bcs = [DirichletBC(V, 0.0, s) for s in ("bottom", "top")]
        L = assemble(mass(V), u=V.dat(np.sin(np.arange(V.node_count) * 0.37)))
        u = V.dat()
        eng.names, eng.trace = [], []
        solve(Form(V), L, u, bcs=bcs, hierarchy=h, solver_parameters=dict(CASES[case], ksp_rtol=1e-14, ksp_max_it=2))
        return list(eng.names), [":".join(str(v) for v in t if v is not None) for t in eng.trace]
