/* fdb200.h -- C ABI of the H100-native (sm_90a) finite-element assembly engine.
 *
 * This is the drop-in boundary for ONE hot path of firedrakeproject/firedrake:
 * the compiled PyOP2 "global kernel" (gather through the cell->node map, run
 * the TSFC element kernel, scatter-add into a Dat or a Mat) and the data
 * movement immediately around it.  Every entry point cites the reference
 * interface it replaces (paths relative to the reference tree).
 *
 * Conventions
 *   - IntType  = int32 (PETSc default; reference pyop2/datatypes.py:5-9)
 *   - ScalarType = double (reference tsfc/parameters.py:18-22)
 *   - all functions return 0 on success, nonzero on failure; the message is
 *     available from fdb_last_error().  The reference wrapper ignores return
 *     codes and raises in Python before the launch (pyop2/parloop.py:175-189);
 *     the Python shim raises on nonzero.
 *   - one CUDA device and one stream per process (one process per GPU).
 *   - plain pointers and sizes only; no torch / PETSc types.
 */
#ifndef FDB200_H
#define FDB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef int32_t fdb_int;

/* ------------------------------------------------------------------ runtime */
/* Select the device and create the engine stream.  Idempotent.  Replaces the
 * implicit "cc + dlopen" environment of pyop2/compilation.py:424-455. */
int fdb_init(int device);
int fdb_finalize(void);
const char *fdb_last_error(void);
int fdb_synchronize(void);
/* name, SM count, total memory of the active device */
int fdb_device_info(char *name, int name_len, int *sm_count, size_t *total_mem);
/* number of kernels this library has launched since fdb_init (bench.py's
 * "gpu_launches" claim is read from here, not estimated) */
uint64_t fdb_launch_count(void);

/* Engine options (kernel selection knobs; each also has an environment default):
 *   "matrix_kernel"  -1 auto (dense B^T D B on the fp64 tensor pipe for degrees 3 and 4, the
 *                       sum-factorised column kernel otherwise), 0 always sum-factorised, 1 DMMA wherever instantiated
 *                       (degrees 2..4)                                   [env FDB_MATRIX_DMMA]
 * Returns nonzero for an unknown name. */
int fdb_set_option(const char *name, int value);
int fdb_get_option(const char *name, int *value);

/* --------------------------------------------------------- device-resident data
 * Device storage for Dat/Map/Global payloads when the caller keeps data on the
 * GPU across calls (SURVEY.md section 8f row f1).  Layout is exactly the host
 * layout of pyop2/types/dat.py:72-96: C-contiguous (total_size, *dim), owned
 * rows first, ghost rows at the tail, vector spaces AoS. */
void *fdb_malloc(size_t nbytes);
int fdb_free(void *dptr);
int fdb_memset(void *dptr, int value, size_t nbytes);
int fdb_memcpy_h2d(void *dst_dev, const void *src_host, size_t nbytes);
int fdb_memcpy_d2h(void *dst_host, const void *src_dev, size_t nbytes);
int fdb_memcpy_d2d(void *dst_dev, const void *src_dev, size_t nbytes);
/* Zero a buffer on a side stream, ordered after everything already enqueued on
 * the engine stream (the buffer may still be in use there); the engine stream
 * is not blocked.  fdb_background_barrier() makes the engine stream wait for
 * all such zeroing issued so far.  Used to rotate pre-zeroed output buffers so
 * that the assembler's "zero the tensor" (firedrake/assemble.py:1042-1047)
 * overlaps the previous global kernel instead of preceding the next one. */
int fdb_zero_background(void *dptr, size_t nbytes);
int fdb_background_barrier(void);
/* pinned host staging (the e2e path copies from/to these) */
void *fdb_host_alloc(size_t nbytes);
int fdb_host_free(void *hptr);
int fdb_host_register(void *hptr, size_t nbytes);
int fdb_host_unregister(void *hptr);

/* ------------------------------------------------------------- mirror cache
 * Drop-in mode: the caller hands HOST pointers, exactly what
 * pyop2/parloop.py:203-212 puts in the arglist.  The engine keeps a device
 * mirror per (host pointer, nbytes) and re-uploads when `version` differs from
 * the one it holds -- `version` is DataCarrier.dat_version
 * (pyop2/types/data_carrier.py:79-97), bumped by the caller on every host
 * write.  FDB_WRITEBACK copies the mirror back to the host buffer. */
int fdb_mirror_acquire(const void *host, size_t nbytes, uint64_t version,
                       int upload, void **dev_out);
int fdb_mirror_writeback(void *host);
/* partial transfers host <-> mirror (byte offset / length inside the buffer), asynchronous on the
 * engine stream (download: `sync` waits), and the version the mirror is current for */
int fdb_mirror_upload_range(const void *host, size_t offset, size_t nbytes);
int fdb_mirror_download_range(void *host, size_t offset, size_t nbytes, int sync);
int fdb_mirror_set_version(const void *host, uint64_t version);
int fdb_mirror_drop(const void *host);
int fdb_mirror_drop_all(void);

/* ------------------------------------------------------------ global kernels
 * fdb_kernel_desc is what PyOP2 folds into the JIT-compiled wrapper as
 * compile-time constants and therefore into GlobalKernel.cache_key
 * (pyop2/global_kernel.py:309-317): map arities, offset[], dims, extruded,
 * constant_layers, subset, access modes -- plus the identity of the local
 * kernel, which here is a form descriptor instead of generated C (the
 * reference keys its kernel cache on the UFL form signature,
 * firedrake/tsfc_interface.py:55-62). */

enum fdb_form {
    FDB_FORM_HELMHOLTZ = 1,     /* alpha*inner(grad u, grad v)*dx + beta*inner(u, v)*dx;
                                   Poisson: (1,0)  mass: (0,1)  Helmholtz: (1,1)
                                   demos/helmholtz/helmholtz.py.rst:52-77,
                                   demos/matrix_free/poisson.py.rst:13-27        */
    FDB_FORM_DG_ADVECTION = 2,  /* demos/DG_advection/DG_advection.py.rst:182-217 */
    FDB_FORM_HELMHOLTZ_COEF = 3, /* alpha*inner(kappa*grad u, grad v)*dx + beta*inner(u, v)*dx with a
                                   scalar coefficient FIELD kappa in the argument space, gathered
                                   through the same cell->node map (maps[0]); beta stays a constant.
                                   Heterogeneous materials, Newton Jacobians of nonlinear diffusion.
                                   Hex cells (extruded or native), cdim == 1, nq == degree+1,
                                   affine_cells == 0; degrees 1..5 (action), 1..4 (rank 2), 1..3
                                   (diagonal).  kappa is always the LAST argument:
                                     action    [y INC, coords, u, kappa]  (atomic or coloured;
                                               device or host mode, host mode monolithic)
                                     diagonal  [d INC, coords, kappa]     (device mode)
                                     rank 2    [Mat, coords, kappa]
                                   Always the sum-factorised slab-thread kernel: the option
                                   "matrix_kernel" (DMMA element matrices) does not apply.       */
    FDB_FORM_NONLINEAR_DIFFUSION = 4,
                                /* residual of nonlinear diffusion, no source term:
                                     F(u; v) = alpha*inner(D(u) grad u, grad v)*dx + beta*inner(u, v)*dx
                                   D(s) = dcoef[0] + dcoef[1] s + dcoef[2] s^2, evaluated at each
                                   Gauss point from the interpolated u.  Rank 1 action only (not rank
                                   2, not diagonal):  [y INC, coords, u].  Hex cells, cdim == 1,
                                   nq == degree+1, affine_cells == 0, degrees 1..5; atomic or
                                   coloured scatter, device or host mode (host mode monolithic).   */
    FDB_FORM_NONLINEAR_DIFFUSION_JACOBIAN = 5,
                                /* its Gateaux derivative at u (exact Newton Jacobian, NOT symmetric):
                                     J(u)[w; v] = alpha*inner(D(u) grad w + D'(u) w grad u, grad v)*dx
                                                  + beta*inner(w, v)*dx
                                   Same restrictions as FDB_FORM_HELMHOLTZ_COEF, degrees 1..5
                                   (action), 1..4 (rank 2), 1..3 (diagonal).  u is always the LAST
                                   argument, gathered through maps[0]:
                                     action    [y INC, coords, w, u]
                                     diagonal  [d INC, coords, u]      (device mode)
                                     rank 2    [Mat, coords, u]  (row = test dof, column = trial dof)
                                   Never the DMMA element-matrix kernels (they assume symmetry).  */
    FDB_FORM_ELASTICITY = 6,
                                /* linear elasticity on a vector space (value size 3, AoS):
                                     a(u, v) = inner(sigma(u), grad v)*dx + beta*inner(u, v)*dx,
                                     sigma(u) = mu (grad u + grad u^T) + lmbda tr(grad u) I
                                   mu = alpha, beta = beta, lmbda = the field lmbda (dcoef unused).
                                   The components couple: every 3 x 3 block of the element matrix is
                                   filled, and the matrix is symmetric.  Hex cells (extruded or
                                   native), cdim == 3, nq == degree+1, affine_cells == 0; degrees 1..4
                                   (action), 1..3 (rank 2 and diagonal):
                                     action    [y INC, coords, u]  (atomic or coloured; device or host
                                               mode, host mode monolithic)
                                     diagonal  [d INC, coords]     (device mode; 3 values per node)
                                     rank 2    [Mat (block size 3), coords]  (row = test dof,
                                               column = trial dof; dof-level lgmaps)
                                   Never the DMMA element-matrix kernels ("matrix_kernel" does not
                                   apply).                                                          */
    FDB_FORM_HYPERELASTICITY = 7,
                                /* residual of compressible Neo-Hookean hyperelasticity (value size 3):
                                     F = I + grad u,  J = det F,
                                     P(F) = mu (F - F^{-T}) + lmbda ln(J) F^{-T}
                                     R(u; v) = inner(P(F), grad v)*dx + beta*inner(u, v)*dx
                                   mu = alpha, lmbda and beta as for FDB_FORM_ELASTICITY.  J <= 0 at
                                   a Gauss point gives NaN, as ln J does.  Same cells and restrictions
                                   as FDB_FORM_ELASTICITY; rank 1 action only (not rank 2, not
                                   diagonal), degrees 1..4:  [y INC, coords, u]  (atomic or coloured;
                                   device or host mode, host mode monolithic).                      */
    FDB_FORM_HYPERELASTICITY_JACOBIAN = 8,
                                /* its Gateaux derivative at u (exact Newton Jacobian, symmetric):
                                     J(u)[w; v] = inner(dP[grad w], grad v)*dx + beta*inner(w, v)*dx
                                     dP[H] = mu H + (mu - lmbda ln J) F^{-T} H^T F^{-T}
                                             + lmbda tr(F^{-1} H) F^{-T}
                                   Degrees 1..4 (action), 1..3 (rank 2 and diagonal).  u is always
                                   the LAST argument, gathered through maps[0]:
                                     action    [y INC, coords, w, u]  (device or host mode)
                                     diagonal  [d INC, coords, u]     (device mode)
                                     rank 2    [Mat (block size 3), coords, u]                      */
    FDB_FORM_ADVECTION_DIFFUSION = 9,
                                /* advection-diffusion of a scalar (NOT symmetric):
                                     a(u, v) = alpha*inner(grad u, grad v)*dx
                                               + inner(dot(b, grad u), v)*dx + beta*inner(u, v)*dx
                                   b is a vector FIELD of 3 components on the nodes of the scalar
                                   argument space, AoS (node i holds b[3 i + c]), gathered through
                                   maps[0].  Hex cells (extruded or native), cdim == 1, nq ==
                                   degree+1, affine_cells == 0; degrees 1..4 (action), 1..3 (rank 2
                                   and diagonal).  b is always the LAST argument:
                                     action    [y INC, coords, u, b]  (atomic or coloured; device or
                                               host mode, host mode monolithic)
                                     diagonal  [d INC, coords, b]     (device mode)
                                     rank 2    [Mat, coords, b]  (row = test dof, column = trial dof)
                                   Never the DMMA element-matrix kernels (they assume symmetry).  */
    FDB_FORM_STOKES = 10,
                                /* Stokes flow on Taylor-Hood hexahedra: velocity u in vector CG_p
                                   (value size 3, AoS, maps[0]) and pressure p in scalar CG_{p-1}
                                   (one value per node, maps[2]) on the same cells,
                                     a((u, p), (v, q)) = mu*inner(grad u, grad v)*dx
                                                         + beta*inner(u, v)*dx
                                                         - p*div(v)*dx - q*div(u)*dx
                                   mu = alpha, beta = beta (beta = 1/dt: an implicit Euler step of
                                   unsteady Stokes).  Symmetric and indefinite; the pressure rows carry
                                   -q div u (Firedrake's Stokes demo writes +q div u: the same system
                                   with the pressure rows negated).  degree = p (2..4), cdim == 3,
                                   nq == p+1, affine_cells == 0, B/D the velocity tables.  A form on
                                   two spaces: created by fdb_kernel_create_mixed, whose
                                   fdb_space2_desc gives the pressure space (degree p-1, its basis at
                                   the nq Gauss points and, on extruded cells, the pressure map's
                                   layer offsets).  Rank 1 action only (not rank 2, not diagonal),
                                   device mode only, atomic or coloured scatter:
                                     action  [y_u INC, coords, u, y_p INC, p]
                                             maps [V map, coord map, Q map]                       */
    FDB_FORM_NAVIER_STOKES = 11,
                                /* residual of steady incompressible Navier-Stokes on the Taylor-Hood
                                   spaces of FDB_FORM_STOKES (NOT symmetric):
                                     R((u, p); (v, q)) = nu*inner(grad u, grad v)*dx
                                                         + beta*inner(u, v)*dx
                                                         + inner(dot(grad u, u), v)*dx
                                                         - p*div(v)*dx - q*div(u)*dx
                                   nu = alpha, dot(grad u, u)_d = sum_k du_d/dx_k u_k.  The Stokes sign
                                   convention: R at u = 0 is the Stokes action.  Same spaces, creation
                                   (fdb_kernel_create_mixed) and restrictions as FDB_FORM_STOKES; the
                                   convective term is not integrated exactly by the nq = p+1 rule.
                                     action  [y_u INC, coords, u, y_p INC, p]
                                             maps [V map, coord map, Q map]                       */
    FDB_FORM_NAVIER_STOKES_JACOBIAN = 12,
                                /* its Gateaux derivative at the velocity u (exact Newton Jacobian, NOT
                                   symmetric), applied to the direction (w, r):
                                     J(u)[(w, r); (v, q)] = nu*inner(grad w, grad v)*dx
                                                            + beta*inner(w, v)*dx
                                                            + inner(dot(grad w, u), v)*dx
                                                            + inner(dot(grad u, w), v)*dx
                                                            - r*div(v)*dx - q*div(w)*dx
                                   J at u = 0 is FDB_FORM_STOKES.  Same restrictions as FDB_FORM_STOKES.
                                   The second space's arguments come first, then u, always the LAST
                                   argument, read through maps[0]:
                                     action  [y_u INC, coords, w, y_p INC, r, u]
                                             maps [V map, coord map, Q map]                       */
    FDB_FORM_BOUNDARY_MASS = 13,
                                /* the boundary mass term, an EXTERIOR-FACET integral (symmetric):
                                     a(u, v) = gamma*inner(u, v)*ds
                                   gamma = alpha.  The Robin operator term, and through its action every
                                   boundary load: inner(g, v)*ds is the action on g with gamma = 1 (a
                                   Neumann flux for scalar g, a traction for vector g).  integral ==
                                   FDB_INTEGRAL_EXTERIOR_FACET (cell and interior-facet integrals are
                                   refused).  Hex cells (extruded or native), cdim 1 or 3, nq ==
                                   degree+1, affine_cells == 0; degrees 1..5 (action and diagonal), 1..4
                                   (rank 2).  An iteration entry is one facet of one cell: the maps are
                                   the owning cell's rows (plus offset * layer on extruded cells), and the
                                   LAST argument is a uint32 local facet number per entry (per column on
                                   extruded sets), 2*direction + side: 0 / 1 where the x dof index of the
                                   local numbering (ax*N + ay)*N + az is 0 / 1, 2 / 3 for y, 4 / 5 for z
                                   (bottom / top).  Device mode only:
                                     action    [y INC, coords, u, facet]  (atomic or coloured)
                                     diagonal  [d INC, coords, facet]     (cdim values per node, the
                                               same in each component)
                                     rank 2    [Mat, coords, facet]  (block size cdim; the components
                                               do not couple: block diagonals only)               */
    FDB_FORM_INTERIOR_PENALTY = 14,
                                /* the interior-facet terms of the symmetric interior penalty (SIPG)
                                   discretisation on scalar DQ_p (Gauss-Legendre nodes), an
                                   INTERIOR-FACET integral (symmetric):
                                     a(u, v) = alpha*( -inner(avg(grad u), jump(v, n))
                                                       - inner(jump(u, n), avg(grad v))
                                                       + (eta/avg(h))*inner(jump(u, n), jump(v, n)) )*dS
                                   alpha = alpha, eta = beta; h = the cell diameter (largest distance
                                   between two of the cell's 8 vertices), n the unit normal outward from
                                   '+'.  integral == FDB_INTEGRAL_INTERIOR_FACET.  Hex cells (extruded or
                                   native), cdim 1, nq == degree+1, affine_cells == 0, degrees 1..4,
                                   action and diagonal (there is no assembled DG matrix: rank 2 is
                                   refused).  An iteration entry is one facet: maps[0] is the '+' cell's
                                   row followed by the '-' cell's (arity 2*(degree+1)^3, offsets tiled),
                                   maps[1] their 8 + 8 vertices; the LAST argument holds the two uint32
                                   local facet numbers ('+', '-') of each entry (per column on extruded
                                   sets, numbered as for FDB_FORM_BOUNDARY_MASS).  Both sides must
                                   parametrise the face alike: face point (s, t) of '+' is face point
                                   (s, t) of '-'.  Device mode only:
                                     action    [y INC, coords, u, facets]  (atomic or coloured)
                                     diagonal  [d INC, coords, facets]                            */
    FDB_FORM_DG_BOUNDARY = 15,
                                /* the exterior-facet terms of the same discretisation, an
                                   EXTERIOR-FACET integral:
                                     a(u, v) = ( c_m*u*v + (c_p/h)*u*v - c_s*u*dot(grad v, n)
                                                 - c_f*dot(grad u, n)*v )*ds
                                   c_f = alpha, c_p = beta, c_m = dcoef[0], c_s = dcoef[1].  Nitsche's
                                   weak Dirichlet operator is (c_m, c_p, c_s, c_f) = (0, alpha*eta,
                                   alpha, alpha); its action on g with (0, alpha*eta, alpha, 0) is the
                                   Dirichlet load of g, with (1, 0, 0, 0) the flux load g*v*ds.  Hex
                                   cells, cdim 1, nq == degree+1, affine_cells == 0, degrees 1..4,
                                   action and diagonal (rank 2 is refused).  An iteration entry is one
                                   facet of one cell: the cell's rows (full (degree+1)^3 and 8), the LAST
                                   argument its uint32 local facet number.  Device mode only:
                                     action    [y INC, coords, u, facet]  (atomic or coloured)
                                     diagonal  [d INC, coords, facet]                             */
    FDB_FORM_DG_TRANSPORT = 16,
                                /* upwind DG transport of a scalar DQ_p field (Gauss-Legendre nodes) by
                                   a velocity b given at the mesh VERTICES (3 values per vertex, read
                                   through maps[1], the vertex map), in conservative form (NOT
                                   symmetric).  The integral selects the term:
                                     cell            - u*dot(b, grad v)*dx
                                     interior facet  dot(b, n('+'))*u_up*(v('+') - v('-'))*dS,
                                                     u_up = u('+') if b.n >= 0 else u('-')
                                     exterior facet  (c_out*max(b.n, 0) + c_in*min(b.n, 0))*u*v*ds
                                   c_out = dcoef[0], c_in = dcoef[1] (the outflow operator is (1, 0),
                                   the inflow load of g the action on g with (0, -1)).  b is the
                                   trilinear interpolant of the vertex values; n and the face weight
                                   are the '+' side's, applied with opposite signs to the two sides, so
                                   1^T A q is exactly the outflow flux.  Hex cells, cdim 1, degrees
                                   1..4, action and diagonal (rank 2 is refused: there is no assembled
                                   DG matrix).  The collocated GL element only: B must be the identity
                                   and nq == degree+1.  Facet entries and maps as for
                                   FDB_FORM_INTERIOR_PENALTY / FDB_FORM_DG_BOUNDARY; a cell entry's
                                   dofs must belong to that cell alone (a DQ map), since the cell
                                   kernel adds into y without atomics.  Device mode only:
                                     cell      action    [y INC, coords, u, b]
                                               diagonal  [d INC, coords, b]
                                     facets    action    [y INC, coords, u, b, facets]  (atomic or
                                                                                         coloured)
                                               diagonal  [d INC, coords, b, facets]               */
    FDB_FORM_P_PROLONG = 17,
    FDB_FORM_P_RESTRICT = 18,
    FDB_FORM_P_INJECT = 19,
                                /* the degree transfers of p-multigrid between a fine space CG_p and a
                                   coarse space CG_q on the SAME hex cells, both on GLL nodes (value size
                                   cdim 1 or 3, AoS), cell-local and sum-factorised:
                                     P_PROLONG   fine    = (P (x) P (x) P) coarse           WRITE
                                     P_RESTRICT  coarse += (P (x) P (x) P)^T (w o fine)     INC
                                     P_INJECT    coarse  = (R (x) R (x) R) fine             WRITE
                                   Tables, row-major in 1-D dof numbering (dof 0 at x = 0, dof 1 at x = 1,
                                   then the interior nodes):
                                     P (p+1, q+1), the coarse basis at the fine nodes: fdb_space2_desc.B
                                     R (q+1, p+1), the fine basis at the coarse nodes: fdb_kernel_desc.B,
                                                   with nq = q+1
                                   The descriptor describes the fine space (degree = p, cdim, offset0 = the
                                   fine map's layer offsets; offset1, D, wq, xq unused), fdb_space2_desc the
                                   coarse space (degree = q, offset = the coarse map's layer offsets).
                                   Created by fdb_kernel_create_mixed, rank 1, cell integral.  (p, q) in
                                   {(2, 1), (3, 1), (3, 2)}.  The endpoint rows (dofs 0 and 1) of P and R
                                   must be exact unit vectors, as they are for GLL elements (a Gauss-Legendre,
                                   DQ, element is refused): every cell that writes a shared node then
                                   writes bitwise the same value.  w is one value per fine node, 1 / (number
                                   of cells containing it), so that the restriction is exactly P^T.  The
                                   maps are in first-use order of the arguments.  Device mode only:
                                     P_PROLONG   [fine WRITE, coarse]       maps [fine map, coarse map]
                                     P_RESTRICT  [coarse INC, fine, w]      maps [coarse map, fine map]
                                                                            (atomic or coloured scatter;
                                                                            coloured is bit-reproducible)
                                     P_INJECT    [coarse WRITE, fine]       maps [coarse map, fine map]  */
    FDB_FORM_SPECTRAL_HELMHOLTZ = 20,
    FDB_FORM_SPECTRAL_HELMHOLTZ_COEF = 21,
                                /* the spectral-element (SEM) Helmholtz operator on scalar CG_p, integrated
                                   with the GLL rule at the nodes themselves (mass lumping):
                                     alpha*inner(kappa*grad u, grad v)*dx(GLL) + beta*inner(u, v)*dx(GLL)
                                   kappa = 1 for SPECTRAL_HELMHOLTZ; SPECTRAL_HELMHOLTZ_COEF reads a
                                   nodal kappa (c^2 of the wave equation) through maps[0].  The tables
                                   are the GLL rule in dof order: nq == degree+1, xq = the nodes (xq[0]
                                   == 0, xq[1] == 1 exactly), B exactly the identity, D the GLL
                                   differentiation matrix D[q][a] = l_a'(x_q).  The mass term is then
                                   diagonal, beta*w_i*|det J_i| at node i.  Trilinear geometry.  Hex cells
                                   (extruded or native), cdim 1, affine_cells 0, degrees 1..5, action
                                   and diagonal at every degree; rank 2 is refused (there is no
                                   assembled SEM matrix).  Device mode only, atomic or coloured scatter
                                   (coloured is bit-reproducible):
                                     action    [y INC, coords, u]            SPECTRAL_HELMHOLTZ
                                               [y INC, coords, u, kappa]     SPECTRAL_HELMHOLTZ_COEF
                                     diagonal  [d INC, coords]               SPECTRAL_HELMHOLTZ
                                               [d INC, coords, kappa]        SPECTRAL_HELMHOLTZ_COEF      */
    FDB_FORM_MIXED_POISSON = 22,
                                /* mixed Poisson / Darcy on the H(div) pair NCF_k x DQ_{k-1} (k = 2..4; Firedrake's
                                   "spectral" variants), symmetric and indefinite:
                                     a((sigma, u), (tau, v)) = alpha*dot(sigma, tau)*dx + div(tau)*u*dx
                                                               + div(sigma)*v*dx
                                   A flux dof is one component of sigma^ = det J J^-1 sigma (the contravariant Piola
                                   pull-back) at its node; component d is CG_k on GLL nodes along axis d and DG_{k-1}
                                   on Gauss-Legendre nodes along the other two.  Local numbering component-major,
                                   block d index (i0*n1 + i1)*n2 + i2 with n_d = k+1, n_e = k, the CG index in 1-D dof
                                   numbering (0 at 0, 1 at 1, then the interior): arity 3 k^2 (k+1).  The descriptor
                                   is NCF_k: degree k, cdim 1, nq == k+1, B / D the CG_k tables at the Gauss points,
                                   offset0 the NCF map's layer offsets; fdb_space2_desc is DQ_{k-1}: degree k-1, B its
                                   Gauss-Legendre basis at the same points (nq, k), offset the DQ map's.  det J > 0 is
                                   assumed (the Piola identities then take det J out of B).  Rank 1 only, affine_cells
                                   0, created by fdb_kernel_create_mixed; device mode, atomic or coloured scatter
                                   (coloured is bit-reproducible), extruded and native hexes:
                                     action    [y_sigma INC, coords, sigma, y_u INC, u]
                                               maps [NCF map, coord map, DQ map]
                                               y_sigma += alpha M sigma + B^T u,  y_u += B sigma
                                     diagonal  [d INC, coords]   maps [NCF map, coord map]
                                               d += diag(alpha M), one value per flux dof               */
    FDB_FORM_MIXED_POISSON_SCHUR = 23,
                                /* the selfp Schur complement of FDB_FORM_MIXED_POISSON, S_p = B W B^T with W a
                                   diagonal given as one value per flux dof (diag(alpha M)^-1, zero on flux-condition
                                   rows).  Metric-free: no coordinates.  Same descriptor, second space, restrictions
                                   and creation as FDB_FORM_MIXED_POISSON (alpha is not read):
                                     action    [y_u INC, u, w, t INC]   maps [DQ map, NCF map]
                                               t += B^T u (over the cells), then y_u += B (w o t) (a second pass):
                                               y_u += S_p u when t is zero on entry
                                     diagonal  [d INC, w]   maps [DQ map, NCF map]
                                               d += diag(B W B^T), one pass                            */
    FDB_FORM_BOUSSINESQ = 24,
                                /* residual of the Boussinesq (Rayleigh-Benard) system on the Taylor-Hood spaces
                                   of FDB_FORM_STOKES with a temperature T in scalar CG_{p-1} on the PRESSURE
                                   numbering (one value per node of maps[2]; NOT symmetric):
                                     R((u, p, T); (v, q, S)) = nu*inner(grad u, grad v)*dx + beta*inner(u, v)*dx
                                                               + inner(dot(grad u, u), v)*dx
                                                               - p*div(v)*dx - T*inner(bg, v)*dx
                                                               - q*div(u)*dx
                                                               + dot(grad T, u)*S*dx
                                                               + kT*inner(grad T, grad S)*dx
                                   nu = alpha, bg = dcoef[0..2] (the buoyancy vector (Ra/Pr) g), kT = lmbda
                                   (1/Pr).  The (u, p) rows are FDB_FORM_NAVIER_STOKES when bg = 0.  The
                                   convective terms are not integrated exactly by the nq = p+1 rule.  Same
                                   spaces, creation (fdb_kernel_create_mixed, the pressure space as the second
                                   space) and restrictions as FDB_FORM_STOKES:
                                     action  [y_u INC, coords, u, y_p INC, p, y_T INC, T]
                                             maps [V map, coord map, Q map]                       */
    FDB_FORM_BOUSSINESQ_JACOBIAN = 25,
                                /* its Gateaux derivative at (u0, T0) (exact Newton Jacobian, NOT symmetric),
                                   applied to the direction (w, r, s):
                                     J[(w, r, s); (v, q, S)] = FDB_FORM_NAVIER_STOKES_JACOBIAN at u0 on (w, r)
                                                               - s*inner(bg, v)*dx
                                                               + dot(grad s, u0)*S*dx + dot(grad T0, w)*S*dx
                                                               + kT*inner(grad s, grad S)*dx
                                   Parameters and restrictions as FDB_FORM_BOUSSINESQ.  The linearisation point
                                   comes LAST: u0 through maps[0], T0 through maps[2]:
                                     action  [y_u INC, coords, w, y_p INC, r, y_T INC, s, u0, T0]
                                             maps [V map, coord map, Q map]                       */
    FDB_FORM_MIXED_POISSON_HYBRID = 26,
    FDB_FORM_MIXED_POISSON_RECONSTRUCT = 27,
                                /* hybridisation of FDB_FORM_MIXED_POISSON (k = 2..3): the flux space broken cell by
                                   cell, normal continuity enforced by lambda in the HDiv-trace space (Q_{k-1} on each
                                   face, k^2 dofs at its Gauss-Legendre points; local numbering face 2d + s, then
                                   t0 * k + t1 with the two GL indices in axis order: 6k^2 per cell).  With K_K the
                                   cell's [[alpha M, B^T], [B, 0]] and C^ = [C 0], C[t][sigma-dof(t)] = o_t w_t0 w_t1
                                   (o = -1 on side s = 0, +1 on s = 1; w the k-point GL weights):
                                     H = sum_K C^ K_K^-1 C^^T   (symmetric positive semi-definite)
                                     r = sum_K C^ K_K^-1 f_K,   (sigma_K, u_K) = K_K^-1 (f_K - C^^T lambda)
                                   f_K = (w o f_sigma, f_u) gathered through the NCF and DQ maps, w one value per
                                   flux dof.  Descriptor, second space and creation (fdb_kernel_create_mixed) as
                                   FDB_FORM_MIXED_POISSON, except that offset0 holds the trace map's 6k^2 layer
                                   offsets FOLLOWED by the NCF map's 3k^2(k+1) (offset1 the coordinate map's, the
                                   second space's offset the DQ map's).  Degree 4 is refused (its local flux mass
                                   matrix exceeds the shared memory of an SM).  Device mode, atomic scatter only
                                   (every entry receives at most two cell contributions: bit-reproducible), extruded
                                   and native hexes, no diagonal:
                                     HYBRID       rank 2  [H mat INC, coords]   maps [trace map, coord map]
                                                          H += H_K through the Mat's lgmaps (masked rows and
                                                          columns are skipped)
                                                  rank 1  [r INC, coords, f_sigma, w, f_u]
                                                          maps [trace map, coord map, NCF map, DQ map]
                                     RECONSTRUCT  rank 1  [y_sigma INC, coords, lambda, f_sigma, w, y_u INC, f_u]
                                                          maps [NCF map, coord map, trace map, DQ map]
                                                          y_sigma += w o sigma_K, y_u += u_K               */
    FDB_FORM_TRACE_PROLONG = 28,
    FDB_FORM_TRACE_RESTRICT = 29,
                                /* the transfers between CG1 (vertex values) and the HDiv-trace space of
                                   FDB_FORM_MIXED_POISSON_HYBRID (k = 2, 3) on the SAME hex cells, the level transfers
                                   of the two-level GTMG cycle for the trace system, cell-local and metric-free:
                                     TRACE_PROLONG   lambda  = P c                 WRITE
                                     TRACE_RESTRICT  c      += P^T (w o lambda)    INC
                                   Trace dof t (face 2d + s, GL indices t0, t1 along the tangential axes in axis
                                   order) takes the value at its face point of the trilinear interpolant of the cell's
                                   8 vertex values (CG1 local vertex (a0 * 2 + a1) * 2 + a2).  w is one value per trace
                                   dof, 1 / (number of cells holding it), so that the restriction is exactly P^T.
                                   The descriptor describes the trace space: degree = k - 1 (1 or 2), nq = k, cdim 1,
                                   offset0 = the trace map's 6k^2 layer offsets (B, D, wq, xq, offset1 unused);
                                   fdb_space2_desc is CG1: degree 1, B = the CG1 basis at the k Gauss-Legendre points,
                                   (k, 2), offset = the CG1 map's 8 layer offsets.  Created by fdb_kernel_create_mixed,
                                   rank 1, cell integral; other degrees, other second spaces, rank 2 and the diagonal
                                   are refused.  Prolong: every cell sharing a face writes its dofs, each summing its
                                   four vertex terms in ascending order of the global vertex number, so both writers
                                   store bitwise the same value (whatever the local vertex order of either cell).  The
                                   maps are in first-use order of the arguments.  Device mode only, extruded and native
                                   hexes:
                                     TRACE_PROLONG   [lambda WRITE, c]        maps [trace map, CG1 map]
                                     TRACE_RESTRICT  [c INC, lambda, w]       maps [CG1 map, trace map]
                                                                              (atomic or coloured scatter, coloured
                                                                              on the CG1 map: bit-reproducible)   */
};

enum fdb_cell {
    FDB_CELL_HEX_EXTRUDED = 1,  /* quad base mesh x layers: map per column + offset */
    FDB_CELL_HEX = 2,           /* native hex mesh: one map row per cell, no offset  */
    FDB_CELL_TRIANGLE = 3,      /* affine P1 triangles (config 1)                     */
    FDB_CELL_QUAD = 4           /* quads (DG advection)                               */
};

enum fdb_integral {
    FDB_INTEGRAL_CELL = 0,
    FDB_INTEGRAL_EXTERIOR_FACET = 1,
    FDB_INTEGRAL_INTERIOR_FACET = 2,
    FDB_INTEGRAL_FUSED = 3      /* DG advection only: cell + all facet integrals of a cell in one
                                   owner-computes pass (no atomics).  args = [out, coords, q, u,
                                   consts, neighbour facet numbers uint32 (ncells,4),
                                   neighbour cells int32 (ncells,4), -1 = boundary]          */
};

enum fdb_scatter {
    FDB_SCATTER_ATOMIC = 0,     /* atomicAdd(double); run-to-run order varies      */
    FDB_SCATTER_COLOURED = 1    /* deterministic: conflict-free colours, no atomics */
};

#define FDB_MAX_1D 8

typedef struct fdb_kernel_desc {
    int32_t form;               /* enum fdb_form                                  */
    int32_t rank;               /* 1: 1-form / action (Dat INC)   2: 2-form (Mat) */
    int32_t cell;               /* enum fdb_cell                                  */
    int32_t integral;           /* enum fdb_integral                              */
    int32_t degree;             /* polynomial degree p of the argument space      */
    int32_t nq;                 /* 1-D quadrature points (hex kernels: == p+1)    */
    int32_t cdim;               /* value size of the argument space (AoS)         */
    int32_t scatter;            /* enum fdb_scatter                               */
    double alpha, beta;
    /* 1-D tables in 1-D dof numbering, row-major (nq, p+1); weights and points
     * on [0,1].  Runtime inputs: the reference gets them from FInAT at kernel
     * generation time (tsfc/fem.py:330-333, 380-391). */
    double B[FDB_MAX_1D * FDB_MAX_1D];
    double D[FDB_MAX_1D * FDB_MAX_1D];
    double wq[FDB_MAX_1D];
    double xq[FDB_MAX_1D];
    /* extruded layer offsets (Map.offset, pyop2/types/map.py:36-56): arity
     * entries for the argument map, 8 for the Q1 coordinate map.  NULL for
     * non-extruded cells.  Copied at creation. */
    const fdb_int *offset0;
    const fdb_int *offset1;
    /* rank 1 only: assemble the DIAGONAL of the bilinear form, A[i] += a(phi_i, phi_i)
     * (assemble(a, diagonal=True), firedrake/assemble.py:1226-1241,
     * tsfc/kernel_interface/common.py:560-570; ImplicitMatrixContext.getDiagonal).
     * args = [d (INC), coords], maps as for a 1-form. */
    int32_t diagonal;
    /* rank 1, hex cells: the caller's PROMISE that every cell is a parallelepiped (constant
     * Jacobian), e.g. an un-warped box mesh.  The kernel then forms the metric once per cell
     * instead of at every quadrature point (about a third fewer fp64 operations at p = 3).
     * TSFC has no such path for tensor-product cells (their coordinate element is not affine,
     * tsfc/fem.py:793-797 unrolls only simplices); fdb_cells_are_affine() checks the promise. */
    int32_t affine_cells;
    /* FDB_FORM_NONLINEAR_DIFFUSION[_JACOBIAN]: D(s) = dcoef[0] + dcoef[1] s + dcoef[2] s^2.
     * FDB_FORM_DG_BOUNDARY: c_m = dcoef[0], c_s = dcoef[1].
     * FDB_FORM_DG_TRANSPORT (exterior facets): c_out = dcoef[0], c_in = dcoef[1].
     * FDB_FORM_BOUSSINESQ[_JACOBIAN]: the buoyancy vector (Ra/Pr) g = dcoef[0..2].
     * Ignored by every other form (a zeroed descriptor stays valid for them). */
    double dcoef[3];
    /* FDB_FORM_ELASTICITY, FDB_FORM_HYPERELASTICITY[_JACOBIAN]: the Lame parameter lambda (mu is
     * alpha).  FDB_FORM_BOUSSINESQ[_JACOBIAN]: the temperature diffusivity 1/Pr.  Ignored by every other
     * form. */
    double lmbda;
} fdb_kernel_desc;

/* The second space of a form on two spaces (FDB_FORM_STOKES, FDB_FORM_NAVIER_STOKES[_JACOBIAN],
 * FDB_FORM_BOUSSINESQ[_JACOBIAN]: the pressure space, which also numbers the temperature), passed to
 * fdb_kernel_create_mixed next to the descriptor of the first (argument) space, which keeps its
 * layout.  degree: the second space's polynomial degree (Stokes: the velocity degree minus 1);
 * B: its basis at the descriptor's nq Gauss points, row-major (nq, degree+1), 1-D dof numbering;
 * offset: the extruded layer offsets of the second space's map, (degree+1)^3 entries, NULL for
 * native hexes, copied at creation.  The p-multigrid transfers (FDB_FORM_P_PROLONG, _RESTRICT, _INJECT)
 * describe their coarse space CG_q here: degree = q and B = P, (fine degree + 1, q + 1); the trace transfers
 * (FDB_FORM_TRACE_PROLONG, _RESTRICT) their CG1 space: degree = 1 and B = the CG1 basis at the k trace points. */
typedef struct fdb_space2_desc {
    int32_t degree;
    double B[FDB_MAX_1D * FDB_MAX_1D];
    const fdb_int *offset;
} fdb_space2_desc;

typedef struct fdb_kernel_s *fdb_kernel_t;

/* Replaces pyop2.global_kernel.compile_global_kernel (global_kernel.py:426-456):
 * "compile" = validate the descriptor, precompute tables, pick the sm_90a
 * kernel instantiation.  Fails (nonzero) for forms outside the supported set. */
int fdb_kernel_create(const fdb_kernel_desc *desc, fdb_kernel_t *out);
/* The same for a form on two spaces (FDB_FORM_STOKES, FDB_FORM_NAVIER_STOKES[_JACOBIAN],
 * FDB_FORM_BOUSSINESQ[_JACOBIAN], the p-multigrid transfers FDB_FORM_P_*, FDB_FORM_MIXED_POISSON[_SCHUR]), which
 * fdb_kernel_create refuses; a form on one
 * space is refused here. */
int fdb_kernel_create_mixed(const fdb_kernel_desc *desc, const fdb_space2_desc *space2, fdb_kernel_t *out);
int fdb_kernel_destroy(fdb_kernel_t k);

/* 1 in *result iff every hex cell of columns [start, end) x nlay layers is a parallelepiped,
 * i.e. the four trilinear terms of its coordinate field are EXACTLY zero (device pointers;
 * off1_host = the 8 layer offsets of the coordinate map or NULL for native hexes). */
int fdb_cells_are_affine(const double *coords, const fdb_int *map1, const fdb_int *off1_host,
                         fdb_int start, fdb_int end, int nlay, int *result);

#define FDB_LOC_HOST 0          /* args/maps are host pointers (mirror cache)      */
#define FDB_LOC_DEVICE 1        /* args/maps are device pointers from fdb_malloc   */

typedef struct fdb_call_args {
    fdb_int start, end;         /* half-open range into the iteration set          */
    const fdb_int *layers;      /* HOST int[2] {bottom, top node layer}, extruded
                                   constant layers (pyop2/types/set.py:336-345);
                                   variable layers (fdb_wrapper_desc.variable_layers):
                                   HOST int[layers_count][2], one row per column;
                                   NULL otherwise                                   */
    const fdb_int *subset;      /* subset indices (same location as args) or NULL  */
    int32_t nargs;              /* TSFC argument order: output, coords, coefficients */
    void *const *args;
    const size_t *arg_bytes;    /* host mode: byte size of each arg buffer          */
    const uint64_t *arg_versions; /* host mode: dat_version per arg, NULL = always upload */
    int32_t nmaps;              /* distinct maps, first-use order                   */
    const fdb_int *const *maps;
    const size_t *map_bytes;    /* host mode                                        */
    int32_t location;           /* FDB_LOC_HOST | FDB_LOC_DEVICE                    */
    int32_t writeback;          /* host mode: copy the output Dat back when done;
                                   the engine then records arg_versions[0]+1 for it,
                                   matching the dat_version bump PyOP2 applies to
                                   written args (pyop2/parloop.py:262-272)           */
    int32_t output_is_zero;     /* host mode: the caller has just zeroed the output
                                   (firedrake/assemble.py:1042-1047), so the mirror
                                   is memset on the device instead of uploaded       */
    const uint64_t *map_versions; /* host mode: a GENERATION id per map (unique per Map object,
                                   never reused): a new Map that happens to live at a freed
                                   Map's address misses the mirror / colouring / pipeline
                                   caches.  NULL = 0 for every map (address-keyed only)      */
    uint64_t subset_version;    /* same for the subset index array                            */
    fdb_int layers_count;       /* variable layers: rows of `layers` (= columns of the set incl.
                                   ghosts); 0 for constant layers                              */
    uint64_t layers_version;    /* generation id of the layers array (mirror key), like map_versions */
} fdb_call_args;

/* Replaces the ctypes call fn(start, end, *arglist) of
 * pyop2/global_kernel.py:327-335 (signature: SURVEY.md section 8b,
 * pyop2/codegen/builder.py:962-981).  The output is INCREMENTED (caller
 * zeroes it: firedrake/assemble.py:1042-1047).  Asynchronous on the engine
 * stream in device mode; host mode returns after the writeback. */
int fdb_kernel_call(fdb_kernel_t k, const fdb_call_args *a);

/* ------------------------------------------- generic wrapper builder (A3-A6)
 * Replaces pyop2/codegen/builder.py WrapperBuilder (:702-1008) + rep2loopy + the
 * host C compiler (pyop2/compilation.py:424-455) for ARBITRARY local kernels:
 * the local kernel arrives as C source (what CStringLocalKernel carries,
 * pyop2/local_kernel.py:186-207, and what TSFC/loopy emit), the engine generates
 * the sm_90a global kernel around it -- one thread per (iteration-set entry,
 * layer): pack through the maps, call the local kernel, unpack with the access
 * descriptor's semantics -- and compiles it at run time with NVRTC.  The
 * hand-written kernels behind fdb_kernel_create stay the fast path for the forms
 * they cover; this is the general one.  The generated code is verified on the
 * CPU (NVRTC compile for sm_90a + a host re-compilation of the same generated
 * body against the reference's golden arrays, tests/test_codegen.py) and on the
 * GPU (tests/test_jit_gpu.py).
 *
 * Packing semantics (pyop2/codegen/builder.py:322-429, 215-300, 520-625):
 *   Dat through a Map  t[f][i][c] = dat[(map[n][perm[i]] + offset[i]*(layer-bottom+f))*cdim + c]
 *                      READ/RW/MIN/MAX packs read the Dat, INC/WRITE packs start at zero;
 *                      unpack: INC += (atomic), MIN/MAX (atomic), WRITE/RW plain store
 *   Dat direct         the kernel gets &dat[n*cdim]; on an extruded set the entry belongs to the
 *                      COLUMN (every layer sees the same one): READ passes the pointer, INC and
 *                      WRITE go through a private copy (atomic add / plain store), RW is refused
 *   Global             READ: pointer to the values; INC/MIN/MAX: privatised per
 *                      thread, combined with warp shuffles + one atomic per warp
 *   Mat                zeroed local tensor (nr*rdim, nc*cdim) row-major, added into
 *                      the CSR through the (masked) lgmaps, ADD_VALUES / INSERT_VALUES
 * `f` has extent 2 for interior-horizontal-facet packs (both cells of a facet). */
enum fdb_access { FDB_READ = 1, FDB_WRITE = 2, FDB_RW = 3, FDB_INC = 4, FDB_MIN = 5, FDB_MAX = 6 };
enum fdb_arg_kind { FDB_ARG_DAT = 1, FDB_ARG_GLOBAL = 2, FDB_ARG_MAT = 3 };
enum fdb_dtype { FDB_F64 = 1, FDB_F32 = 2, FDB_I32 = 3, FDB_U32 = 4, FDB_I64 = 5 };
enum fdb_region {               /* pyop2 iteration regions, builder.py:779-800 */
    FDB_REGION_ALL = 0, FDB_REGION_ON_BOTTOM = 1, FDB_REGION_ON_TOP = 2,
    FDB_REGION_ON_INTERIOR_FACETS = 3
};

#define FDB_WRAP_MAX_ARGS 16
#define FDB_WRAP_MAX_MAPS 8
#define FDB_WRAP_MAX_MATS 4

typedef struct fdb_wrapper_arg {
    int32_t kind;               /* enum fdb_arg_kind                                         */
    int32_t access;             /* enum fdb_access                                           */
    int32_t dtype;              /* enum fdb_dtype (Mat: FDB_F64)                             */
    int32_t dim;                /* Dat: values per node; Global: entries; Mat: row block size */
    int32_t dim2;               /* Mat: column block size                                    */
    int32_t map;                /* Dat: slot in the call's map list, -1 = direct; Mat: row map */
    int32_t map2;               /* Mat: column map slot                                      */
    int32_t arity, arity2;      /* arity of map / map2                                       */
    const fdb_int *offset;      /* extruded: `arity` layer offsets of map (copied), else NULL */
    const fdb_int *offset2;     /* Mat column map                                            */
    const fdb_int *permutation; /* PermutedMap (pyop2/types/map.py:232-290): `arity` entries or NULL */
    int32_t interior_horizontal;/* 1: pack layer and layer+1                                  */
    /* periodic extrusion (fdb_wrapper_desc.extruded_periodic; pyop2/codegen/builder.py:34-61,
     * 100-123): `arity` entries, 1 where the dof sits on the TOP of the cell so that the top
     * layer wraps onto the bottom one:
     *   index = map[n][i] + offset[i] * ( (layer - bottom + f + oq[i]) mod L  -  oq[i] mod L ),
     * L = cell layers per column.  NULL = all zero. */
    const fdb_int *offset_quotient;
    const fdb_int *offset_quotient2;   /* Mat column map */
    /* MixedDat (pyop2/types/dat.py:861-, "one pointer per sub-Dat" in the arglist,
     * pyop2/parloop.py:203-212): 1 = this wrapper argument is the NEXT SEGMENT of the previous
     * one -- its pack is appended to the previous argument's local tensor and the local kernel
     * receives ONE pointer for the whole group (indirect Dats of equal access and dtype only). */
    int32_t mixed_continuation;
} fdb_wrapper_arg;

typedef struct fdb_wrapper_desc {
    const char *kernel_source;  /* C source of the local kernel; #include lines are ignored,
                                   PetscScalar/PetscInt/intN_t/restrict are predefined        */
    const char *kernel_name;    /* the wrapper is called wrap_<kernel_name>
                                   (pyop2/global_kernel.py:344-346)                           */
    int32_t nargs;              /* local-kernel argument order                                */
    const fdb_wrapper_arg *args;
    int32_t extruded;           /* iterate layers                                            */
    int32_t subset;             /* n = subset[n]                                             */
    int32_t iteration_region;   /* enum fdb_region                                           */
    int32_t pass_layer_arg;     /* extruded: append the current layer (int, by value) to the
                                   local kernel's arguments (pyop2/global_kernel.py:277-279)  */
    int32_t extruded_periodic;  /* the columns are periodic in the extruded direction
                                   (ExtrudedSet(..., extruded_periodic=True), pyop2/types/set.py) */
    int32_t variable_layers;    /* 1: `layers` is int[ncolumns][2], every column has its own
                                   [bottom, top) node layers and its map row points at ITS bottom
                                   cell (constant_layers == False: pyop2/codegen/builder.py:754-812,
                                   pyop2/types/set.py:336-345)                                  */
} fdb_wrapper_desc;

/* The generated CUDA source (no GPU needed).  Writes at most `cap` bytes incl.
 * the terminator and always reports the full length in *needed. */
int fdb_wrapper_source(const fdb_wrapper_desc *d, char *buf, size_t cap, size_t *needed);
/* Generate + NVRTC-compile for sm_90a into a cubin image (no GPU needed: this
 * is the ahead-of-time / disk-cache path, pyop2/compilation.py:424-455).  The
 * NVRTC log is available from fdb_last_error() on failure.  *needed is the
 * image size; cubin = NULL only queries it, and a following call with the same
 * descriptor copies that same image (the last one is kept: NVRTC's images of one
 * source differ from compilation to compilation).  A non-NULL cubin smaller than
 * the image is an error. */
int fdb_wrapper_compile(const fdb_wrapper_desc *d, void *cubin, size_t cap, size_t *needed);
/* Generate, compile and load; the handle is called with fdb_kernel_call using
 * the same arglist convention: args[] = one pointer per local-kernel argument
 * (Dat: data; Global: HOST pointer to its values, always; Mat: fdb_mat_t),
 * maps[] = the distinct maps in slot order.  Host mode uploads every Dat
 * through the mirror cache and writes every non-READ Dat back. */
int fdb_wrapper_create(const fdb_wrapper_desc *d, fdb_kernel_t *out);

/* --------------------------------------------------------------- matrices
 * Device CSR replacing op2.Sparsity + op2.Mat over PETSc AIJ
 * (pyop2/types/mat.py:27-292, 607-985; pyop2/sparsity.pyx:106-389).
 * fdb_mat_create = Sparsity construction + Mat allocation + zero fill for a
 * square block whose row and column maps are the same cell->node map
 * (`map_host`: HOST (ncolumns, arity) IntType, `offset_host`: extruded layer
 * offsets or NULL, `nlayers`: cells per column, 1 if not extruded).  The
 * diagonal is always allocated.  A rank-2 fdb_kernel_call takes the fdb_mat_t
 * as args[0] where the reference passes the PETSc Mat handle.
 * lgmaps: HOST arrays of nrows entries, identity except -1 on Dirichlet
 * rows/columns (masked LGMaps, firedrake/functionspaceimpl.py:854-926); NULL
 * restores the identity (pyop2/parloop.py:279-314 swaps them per parloop). */
typedef struct fdb_mat_s *fdb_mat_t;
int fdb_mat_create(fdb_int nrows, const fdb_int *map_host, fdb_int ncolumns, int arity,
                   const fdb_int *offset_host, int nlayers, fdb_mat_t *out);
/* Blocked variant for vector-valued spaces (op2.Mat over a DataSet with cdim > 1, PETSc
 * BAIJ: pyop2/types/mat.py:741-804): same NODE pattern, every stored entry is a bs x bs
 * block (row-major), lgmaps are dof-level (nrows*bs entries, so that a Dirichlet condition
 * on one component can be expressed), get_csr returns node-level rowptr/colidx and
 * nnz*bs*bs values.  fdb_mat_create(...) == fdb_mat_create_blocked(..., bs = 1, ...). */
int fdb_mat_create_blocked(fdb_int nrows, const fdb_int *map_host, fdb_int ncolumns, int arity,
                           const fdb_int *offset_host, int nlayers, int bs, fdb_mat_t *out);
int fdb_mat_destroy(fdb_mat_t m);
int fdb_mat_nnz(fdb_mat_t m, long long *nnz, fdb_int *nrows);
int fdb_mat_zero(fdb_mat_t m);
int fdb_mat_set_lgmaps(fdb_mat_t m, const fdb_int *row_lgmap_host, const fdb_int *col_lgmap_host);
/* Mat.set_local_diagonal_entries (pyop2/types/mat.py:897-937) */
int fdb_mat_set_diagonal(fdb_mat_t m, const fdb_int *rows_host, fdb_int n, double value);
/* rows are NODE rows; idx = component to set, -1 = every component (the `idx` argument of
 * set_local_diagonal_entries, pyop2/types/mat.py:897-937) */
int fdb_mat_set_diagonal_blocked(fdb_mat_t m, const fdb_int *rows_host, fdb_int n, double value, int idx);
/* d[r] = A[r][r] into a device array of nrows doubles (0 where the pattern has no diagonal entry), scalar
 * matrices: the Jacobi preconditioner of an assembled operator (HybridizationPC's trace CG) */
int fdb_mat_get_diagonal(fdb_mat_t m, double *d);
/* y = A x on device pointers (cross-check of assembled vs matrix-free action) */
int fdb_mat_mult(fdb_mat_t m, const double *x, double *y);
/* copy the CSR arrays to the host (any pointer may be NULL); rowptr is int64 */
int fdb_mat_get_csr(fdb_mat_t m, long long *rowptr, fdb_int *colidx, double *vals);


/* ------------------------------------------- batched patch solves (section 8f row f4)
 * TinyASM's BlockJacobi on the device (tinyasm/tinyasm.cpp:27-120): patches are dof lists
 * (CSR-like: patch_ptr[npatch+1] offsets into patch_dofs; for a blocked matrix a dof is
 * node*bs + component).  fdb_asm_update = updateValuesPerBlock (extract P[d_p, d_p], invert in
 * place: Gauss-Jordan with partial pivoting, one CTA per patch); fdb_asm_apply = solve
 * (x[d_p] += inv_p b[d_p] for every patch, additive; device pointers). */
typedef struct fdb_asm_s *fdb_asm_t;
int fdb_asm_create(int npatch, const long long *patch_ptr_host, const fdb_int *patch_dofs_host, fdb_asm_t *out);
int fdb_asm_destroy(fdb_asm_t a);
int fdb_asm_update(fdb_asm_t a, fdb_mat_t mat, int *nsingular);
int fdb_asm_apply(fdb_asm_t a, const double *b, double *x);
int fdb_asm_get_blocks(fdb_asm_t a, double *out_host);

/* ------------------------------------------- fast-diagonalisation vertex-star relaxation (DESIGN.md 4.20)
 * z = sum_v R_v^T A_v^-1 R_v r over the vertex stars of an extruded CG_p space (p = 1..5), A_v the separable
 * patch operator alpha*kbar_v*(K(x)M(x)M + M(x)K(x)M + M(x)M(x)K) + beta*M(x)M(x)M applied through its 1-D
 * eigenbases (csrc/fdm_star_hex.cu).
 *   cell_node_map [ncols][(p+1)^3], offset [(p+1)^3]: the extruded cell-node map, DEVICE arrays that the handle
 *   reads but does not copy or own (they must outlive it).  The other arrays are host arrays, copied at create:
 *   vert_cols [nvert][4]: base column of each quadrant sx*2 + sy around a base vertex, -1 where there is none;
 *   star_vert, star_layer [nstar]: a star's base vertex and node layer; stars sorted by colour (parities of the
 *   vertex lattice), colour c holding stars colour_ptr[c] .. colour_ptr[c+1]-1;
 *   star_table [nstar][3]: pool entries of the x, y, z tables; pool [npool][m*m + 3m], m = 2p-1: S (row = star
 *   node, column = mode), eigenvalues, active mask, existence mask.
 * fdb_fdm_star_update sets alpha, beta and kbar_v = mean of kappa (device, NULL: 1) over the star's nodes;
 * fdb_fdm_star_apply overwrites z (device pointers, r != z). */
typedef struct fdb_fdm_star_s *fdb_fdm_star_t;
int fdb_fdm_star_create(int degree, int nz, int ncols, const fdb_int *cell_node_map, const fdb_int *offset,
                        fdb_int node_count, int nvert, const fdb_int *vert_cols, int nstar, const fdb_int *star_vert,
                        const fdb_int *star_layer, const fdb_int *star_table, const long long *colour_ptr, int npool,
                        const double *pool, fdb_fdm_star_t *out);
int fdb_fdm_star_update(fdb_fdm_star_t h, double alpha, double beta, const double *kappa);
int fdb_fdm_star_apply(fdb_fdm_star_t h, const double *r, double *z);
int fdb_fdm_star_destroy(fdb_fdm_star_t h);

/* --------------------------------------------------------- Dat subset ops (K5)
 * DirichletBC.zero / DirichletBC.set on a node subset (firedrake/bcs.py:192-221,
 * pyop2/types/dat.py:297-311).  Device pointers. */
int fdb_dat_zero_nodes(double *dat, int cdim, const fdb_int *nodes, fdb_int n);
int fdb_dat_set_nodes(double *dat, const double *src, int cdim, const fdb_int *nodes, fdb_int n);
int fdb_dat_set_nodes_scalar(double *dat, double value, int cdim, const fdb_int *nodes, fdb_int n);

/* ------------------------------------------------------ Dat vector algebra (K6)
 * pyop2/types/dat.py:354-540 (_op/_iop/inner/axpy/norm).  Device pointers;
 * reductions return through a host double. */
int fdb_vec_axpy(size_t n, double a, const double *x, double *y);            /* y += a x       */
int fdb_vec_aypx(size_t n, double a, const double *x, double *y);            /* y = x + a y    */
int fdb_vec_scale(size_t n, double a, double *x);
int fdb_vec_fill(size_t n, double a, double *x);                              /* x[:] = a: ghost-row reset
                                                                                 of INC/MIN/MAX Dats,
                                                                                 pyop2/types/dat.py:633-636 */
int fdb_vec_dot(size_t n, const double *x, const double *y, double *out);
int fdb_vec_pointwise_mult(size_t n, const double *x, const double *y, double *w);
/* the vector part of one Chebyshev iteration with a diagonal preconditioner, in one pass, given ax = A x:
 *   d = c_d d + c_z dinv o (b - ax);  x += d
 * (c_d == 0: d is not read, the first iteration) */
int fdb_vec_chebyshev(size_t n, double c_d, double c_z, const double *b, const double *ax, const double *dinv,
                      double *d, double *x);
/* one explicit central-difference (leapfrog) step of M u'' = -r with a lumped (diagonal) M, in one pass:
 *   uprev = 2 u - uprev - dt2 minv o r
 * (four reads, one write per entry); the caller then swaps the roles of u and uprev.  A row with minv == 0 and u, uprev
 * zero (a rigid wall) stays zero. */
int fdb_vec_leapfrog(size_t n, double dt2, const double *minv, const double *r, const double *u, double *uprev);
/* compact gather / scatter through a device index list: the VecScatter of a virtual sub-matrix
 * (MatCreateSubMatrixVirtual, the fallback of firedrake/matrix_free/operators.py:380-405) */
int fdb_vec_gather(size_t n, const fdb_int *idx, const double *src, double *dst);   /* dst[j] = src[idx[j]] */
int fdb_vec_scatter(size_t n, const fdb_int *idx, const double *src, double *dst);  /* dst[idx[j]] = src[j] */

/* ------------------------------------------------- block vectors (BV)
 * SLEPc's BVDot and BVMult over columns that are ordinary device Dats: x and y are HOST arrays of device
 * pointers, one per column, over rows [0, n) (the owned rows).  m and k are each in 1..FDB_BV_MAX_COLUMNS; a NULL
 * array, column or host matrix is refused, and fdb_bv_mult refuses any y_j equal to any x_i (no in-place update).
 *   fdb_bv_dot   G[i*k + j] = x_i . y_j               G on the host, m x k row-major; bitwise repeatable for the
 *                                                     same inputs (fixed-order reduction on a grid fixed by n);
 *                                                     n = 0 gives G = 0
 *   fdb_bv_mult  y_j = beta y_j + alpha sum_i x_i Q[i*k + j]   Q on the host, m x k row-major; beta == 0 does not
 *                                                     read y; n = 0 leaves y unchanged */
#define FDB_BV_MAX_COLUMNS 64
int fdb_bv_dot(size_t n, int m, const double *const *x, int k, const double *const *y, double *g_host);
int fdb_bv_mult(size_t n, int k, double *const *y, double beta, double alpha,
                int m, const double *const *x, const double *q_host);

/* ------------------------------------------------------- point evaluation
 * A point x_k inside a cell is given by the nper = (p+1)^3 global node ids idx[k*nper + j] of its cell and the
 * basis weights w[k*nper + j] = phi_j(x_k) (located on the host).  Device pointers; both are bit-reproducible:
 *   fdb_point_eval   out[k] = sum_j w_kj u[idx_kj], summed in j order                  (point evaluation E u)
 *   fdb_point_load   y[idx_kj] += scale * a_k * w_kj                                  (its adjoint E^T a: the load
 *                    sum_k a_k phi_i(x_k) of point sources), every node's sum in k order, even when points share
 *                    nodes.
 * A point with idx[k*nper] < 0 (one not found in the mesh) evaluates to NaN and adds nothing. */
int fdb_point_eval(fdb_int npts, int nper, const fdb_int *idx, const double *w, const double *u, double *out);
int fdb_point_load(fdb_int npts, int nper, const fdb_int *idx, const double *w, const double *a, double scale,
                   double *y);

/* ----------------------------------------------------------- interpolation
 * Dual-evaluation parloop with WRITE access (firedrake/interpolation.py:977-1171):
 * interpolate a Q1 (x) P1 field (cdim components, AoS) into the Q_p (x) P_p
 * space whose 1-D node positions are `nodes_host` (dof numbering, n1d = p+1).
 * Device pointers for data, maps and the two offset arrays (zeros when not
 * extruded); `nlay` cells per column. */
int fdb_interpolate_q1(double *out, const double *src, const fdb_int *map_t, const fdb_int *map_s,
                       const fdb_int *off_t_dev, const fdb_int *off_s_dev, fdb_int ncols, int nlay,
                       int n1d, int cdim, const double *nodes_host);

/* ---------------------------------------------------- communicator and halos
 * One process per GPU.  The NCCL communicator replaces the MPI communicator of
 * pyop2/mpi.py; the 128-byte unique id is created on rank 0 and distributed by
 * the host launcher (torch.distributed / MPI / a file -- plumbing).
 *
 * A halo replaces firedrake.halo.Halo (firedrake/halo.py:87-172): per
 * neighbour, `send` lists the OWNED dofs that are ghosts on that neighbour and
 * `recv` lists MY ghost dofs owned by it (both in the same canonical order on
 * the two sides).  Index arrays are host pointers, copied at creation.
 *   global_to_local  : owner values -> ghost copies      (PetscSF bcast, REPLACE)
 *   local_to_global  : ghost contributions += into owner (PetscSF reduce, SUM)
 * begin() is asynchronous on a communication stream; kernels launched on the
 * engine stream between begin() and end() overlap the exchange
 * (pyop2/parloop.py:250-253). */
int fdb_comm_get_unique_id(char *out128);
int fdb_comm_init(int rank, int nranks, const char *id128);
int fdb_comm_finalize(void);
int fdb_comm_rank(void);
int fdb_comm_size(void);

typedef struct fdb_halo_s *fdb_halo_t;
int fdb_halo_create(int nneigh, const int *ranks, const fdb_int *send_counts,
                    const fdb_int *send_idx, const fdb_int *recv_counts, const fdb_int *recv_idx,
                    int max_cdim, fdb_halo_t *out);
int fdb_halo_destroy(fdb_halo_t h);
int fdb_halo_global_to_local_begin(fdb_halo_t h, double *dat, int cdim);
int fdb_halo_global_to_local_end(fdb_halo_t h, double *dat, int cdim);
int fdb_halo_local_to_global_begin(fdb_halo_t h, double *dat, int cdim);
int fdb_halo_local_to_global_end(fdb_halo_t h, double *dat, int cdim);
/* in-place all-reduce of n doubles on the device, op 0 sum / 1 min / 2 max
 * (pyop2/parloop.py:411-442 Iallreduce of Globals) */
int fdb_allreduce(double *dev, int n, int op);

/* ------------------------------------------------------------------ timing
 * CUDA events on the engine stream (the stream every kernel above is launched
 * on), for bench.py. */
typedef struct fdb_timer_s *fdb_timer_t;
int fdb_timer_create(fdb_timer_t *out);
int fdb_timer_start(fdb_timer_t t);
int fdb_timer_stop(fdb_timer_t t, float *ms_out);   /* records, synchronises, returns elapsed */
int fdb_timer_destroy(fdb_timer_t t);
/* write `nbytes` of a scratch buffer (> L2) to flush the cache between timed
 * iterations */
int fdb_flush_l2(void);

#ifdef __cplusplus
}
#endif
#endif /* FDB200_H */
