"""TEST INFRASTRUCTURE: the engine entry points that the Taylor-Hood solves call, in order, on the Navier-Stokes
mock engine (tests/test_navier_stokes_host_mock.py): a Stokes solve with a lifted velocity condition under each
Schur factorisation, and Newton on the lid-driven cavity with and without the fieldsplit.  The same function
recorded tests/golden/stokes_engine_calls.json from the version before the mixed assembler took a third block
(Boussinesq's temperature)."""
import numpy as np

import test_navier_stokes_gpu as tn
import test_navier_stokes_host_mock as nm

CASES = ("stokes_none", "stokes_diag", "stokes_lower", "stokes_upper", "ns_none", "ns_diag", "ns_lower")


class Recorder(nm.NavierStokesMockEngine):
    """NavierStokesMockEngine that also records the name of every engine entry point called."""

    def __init__(self, oracle):
        super().__init__(oracle)
        self.names = None

    def __getattribute__(self, name):
        if name.startswith("fdb_"):
            names = object.__getattribute__(self, "names")
            if names is not None:
                names.append(name)
        return object.__getattribute__(self, name)


class recording(nm.install):
    def __init__(self, oracle):
        self.engine = Recorder(oracle)


def solve_calls(oracle, case):
    """Entry-point names of one solve on a 3^3 Q2-Q1 cavity (lid velocity on the top, no slip elsewhere), stopped
    after a few iterations."""
    from firedrake_b200.assemble import Stokes, solve, solve_nonlinear
    kind, fact = case.split("_")
    with recording(oracle) as eng:
        mesh, V, Q, F, bcs = tn._cavity(3, 0.2)
        sp = {"ksp_max_it": 4, "ksp_rtol": 1e-14}
        if fact != "none":
            sp.update(pc_type="fieldsplit", pc_fieldsplit_type="schur", pc_fieldsplit_schur_fact_type=fact,
                      fieldsplit_0_pc_type="jacobi", fieldsplit_1_pc_type="jacobi")
        eng.names = []
        if kind == "stokes":
            S = Stokes(V, Q, 0.2)
            L = S.dat(np.zeros((V.node_count, 3)), np.zeros(Q.node_count))
            solve(S, L, S.dat(), bcs=bcs, solver_parameters=sp, nullspace="constant")
        else:
            solve_nonlinear(F, F.dat(), F.dat(), bcs, dict(sp, snes_max_it=2), nullspace="constant")
        return list(eng.names)
